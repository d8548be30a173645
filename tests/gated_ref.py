"""Test helper: an fp64 reference of the gated networks' kernels (ModifiedMLP, ``NetSpec.gated == 1``; PirateNet,
``gated == 2``), evaluated on the exact values the kernels read from the plan's workspace.

A gated plan stores, besides Z_l, Y and Ybar, the output G_l of what follows every hidden layer l (a gate
``G = V + act(Z)(U - V)``, PirateNet's adaptive residual ``X = alpha act(Z) + (1 - alpha) X_prev``, or the embedding
layer's plain ``act_first(Z)``), the embeddings' pre-activations Zu / Zv and their adjoints Zubar / Zvbar, and for a
PirateNet the adjoint Xres carried by the blocks' residual path (``ppsci_b200_plan_stash_offset`` codes 400 + l,
310 .. 314).  A plan created with ``PPSCI_B200_KEEP_ADJOINTS`` set gives every hidden layer's Zbar_l a plane set of its
own (code 500 + l), so that every pass of every layer can be checked after one call:

* forward: Z_l, Zu, Zv and Y from the stored operand (``layer_ref.layer_errors`` with a plain operand and its
  absolute twin); G_l from Z_l, Zu, Zv with the truncated Cauchy product written here per Taylor direction;
* backward: Gbar_l = Zbar_{l+1} W_{l+1}^T (+ Zubar Wu^T + Zvbar Wv^T into an embedding layer 1, + the carried residual
  adjoint), then torch autograd through the same forward expressions gives Zbar_l, each gate's share of Zubar /
  Zvbar (summed over the gates of the call), Xres as the call leaves it and dLoss/d alpha;
* parameter gradients: dW_l / db_l, dWu / dbu / dWv / dbv (operand: the seeds' jets, or G_1 after an embedding layer)
  and dLoss/d omega over every GEMM that read the seeds.

Units as in ``layer_ref``: forward, dW, db, d alpha and d omega componentwise (over the same expression on absolute
values); the adjoint planes (dx, Zubar, Zvbar, Xres) per channel plane against the plane's largest |ref|."""
from __future__ import annotations

import math
import os
from contextlib import contextmanager
from dataclasses import dataclass
from typing import Dict, Optional, Sequence, Tuple

import torch

from oracle import ppsci_oracle as O
from paddlescience_b200.engine.compiler import compile_residuals
from paddlescience_b200.engine.plan import ResidualPlan
from tests.cases import make_net
from tests.layer_ref import (_cw_err, _directions, act_jets, all_layouts, feature_omegas, last_chunk, layer_errors,
                             omega_errors, omega_offset, param_blocks, seed_jets, stash_views)

CODE_ZU, CODE_ZV, CODE_ZUB, CODE_ZVB, CODE_XRES = 310, 311, 312, 313, 314
CODE_G = 400  # + l
CODE_ZBAR_KEEP = 500  # + l, PPSCI_B200_KEEP_ADJOINTS
KEEP_ENV = "PPSCI_B200_KEEP_ADJOINTS"


# ------------------------------------------------------------------------------------------------------------------
# structure of a gated plan (engine.cu: gate_emb, post_kind, the parameter layout of plan_create)
# ------------------------------------------------------------------------------------------------------------------
def emb_of(net) -> int:
    """1 when layer 1 is an embedding layer whose stored output feeds embed_u / embed_v (PirateNet, ModifiedMLP with
    act_first), 0 when the embeddings read the seeds."""
    return 1 if (net.gated == 2 or net.act_first is not None) else 0


def post_kind(net, l: int) -> str:
    """What follows hidden layer l: "emb" (plain act_first), "mix" (PirateNet's adaptive residual) or "gate"."""
    if emb_of(net) and l == 1:
        return "emb"
    return "mix" if (net.gated == 2 and (l - 2) % 3 == 2) else "gate"


def n_blocks(net) -> int:
    return (len(net.widths) - 3) // 3 if net.gated == 2 else 0


@dataclass
class GateParams:
    Wu: slice
    bu: slice
    Wv: slice
    bv: slice
    alpha: slice
    K: int  # fan-in of the embeddings
    H: int  # their fan-out, the gated layers' width


def gate_params(net) -> GateParams:
    """Slices of [... linear layers | Wu | bu | Wv | bv | alpha_0 .. alpha_{B-1} | omega] in the flat vector."""
    off = sum(b.stop for _, b, _ in param_blocks(net.widths)[-1:])
    e = emb_of(net)
    K, H = net.widths[e], net.widths[e + 1]
    sl = []
    for _ in range(2):
        sl += [slice(off, off + K * H), slice(off + K * H, off + K * H + H)]
        off += K * H + H
    return GateParams(sl[0], sl[1], sl[2], sl[3], slice(off, off + n_blocks(net)), K, H)


def act_of(net, l: int) -> str:
    """Activation of linear layer l's output."""
    return net.act_first if (l == 1 and net.act_first is not None) else net.act


# ------------------------------------------------------------------------------------------------------------------
# forward expressions on jets
# ------------------------------------------------------------------------------------------------------------------
def cauchy(a: torch.Tensor, b: torch.Tensor, compiled) -> torch.Tensor:
    """Jets [C, ...] of the product a b: per Taylor direction the truncated Cauchy product of the normalised
    coefficients, (a b)_k = sum_{j=0..k} a_j b_{k-j}, with coefficient 0 (channel 0) shared by every direction."""
    planes = [None] * a.shape[0]
    planes[0] = a[0] * b[0]
    for order, chans in _directions(compiled):
        ch = [0] + chans
        for k in range(1, order + 1):
            planes[ch[k]] = sum(a[ch[j]] * b[ch[k - j]] for j in range(k + 1))
    return torch.stack(planes)


# elu / selu evaluate their negative branch scale alpha (e^z - 1) as scale alpha e^z - scale alpha (jet_math.h): the
# value carries an absolute rounding of order u scale alpha however small it is
_EXP_SHIFT = {"elu": 1.0, "selu": 1.0507009873554804934193349852946 * 1.6732632423543772848170429916717}


def act_abs(act: str, Z: torch.Tensor, compiled) -> torch.Tensor:
    """``layer_ref.act_jets``' absolute twin, plus scale alpha on the value channel of elu / selu where z0 <= 0 (the
    twin of a lone activation value: inside a GEMM the sum over the fan-in dilutes it, in a gate it does not)."""
    A = act_jets(act, Z, compiled, absolute=True)
    if act in _EXP_SHIFT:
        A[0] = A[0] + _EXP_SHIFT[act] * (Z[0] <= 0)
    return A


def _act(act, Z, compiled, absolute):
    return act_abs(act, Z, compiled) if absolute else act_jets(act, Z, compiled)


def gate_expr(act: str, Z, Zu, Zv, compiled, absolute: bool = False) -> torch.Tensor:
    """G = V + act(Z) (U - V), U = act(Zu), V = act(Zv), on jets; ``absolute``: the componentwise twin."""
    Y, U, V = (_act(act, t, compiled, absolute) for t in (Z, Zu, Zv))
    return V + cauchy(Y, U + V if absolute else U - V, compiled)


def mix_expr(act: str, Z, alpha, Xprev, compiled, absolute: bool = False) -> torch.Tensor:
    """X = alpha act(Z) + (1 - alpha) X_prev (X_prev None: X = act(Z)); ``absolute``: the componentwise twin."""
    A = _act(act, Z, compiled, absolute)
    if Xprev is None:
        return A
    if absolute:
        return abs(float(alpha)) * A + abs(1 - float(alpha)) * Xprev.abs()
    return alpha * A + (1 - alpha) * Xprev


# ------------------------------------------------------------------------------------------------------------------
# views
# ------------------------------------------------------------------------------------------------------------------
def gated_views(plan, n: int, last: bool = False, keep: bool = False) -> Dict[str, torch.Tensor]:
    """``layer_ref.stash_views`` plus "G<l>" of every hidden layer, "Zu", "Zv", "Zub", "Zvb", "Xres" (PirateNet) and,
    for a plan created with PPSCI_B200_KEEP_ADJOINTS (``keep``), "Zbar<l>" of every hidden layer."""
    net = plan.compiled.net
    w = net.widths
    L = len(w) - 1
    H = w[emb_of(net) + 1]
    extra = {f"G{l}": (CODE_G + l, w[l]) for l in range(1, L)}
    extra.update({"Zu": (CODE_ZU, H), "Zv": (CODE_ZV, H), "Zub": (CODE_ZUB, H), "Zvb": (CODE_ZVB, H)})
    if net.gated == 2:
        extra["Xres"] = (CODE_XRES, w[1])
    if keep:
        extra.update({f"Zbar{l}": (CODE_ZBAR_KEEP + l, w[l]) for l in range(1, L)})
    return stash_views(plan, n, last=last, extra=extra)


# ------------------------------------------------------------------------------------------------------------------
# errors
# ------------------------------------------------------------------------------------------------------------------
def _plane_err(out: torch.Tensor, ref: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """(max |out - ref|, max |ref|) per channel plane."""
    return (out.double() - ref).abs().flatten(1).amax(1), ref.abs().flatten(1).amax(1)


class _PlaneMax:
    """Running per-plane maxima of |out - ref| and |ref| over point blocks."""

    def __init__(self):
        self.num = self.den = None

    def add(self, out, ref):
        e, m = _plane_err(out, ref)
        self.num = e if self.num is None else torch.maximum(self.num, e)
        self.den = m if self.den is None else torch.maximum(self.den, m)

    def value(self) -> float:
        return float((self.num / self.den.clamp_min(1e-300)).max())


def seeds(plan, views, params, absolute: bool = False) -> torch.Tensor:
    return seed_jets(plan.compiled, views["X"], feature_omegas(plan, params), absolute)


def forward_errors(plan, views: Dict[str, torch.Tensor], params: torch.Tensor) -> Dict[str, float]:
    """Every forward pass: "fwd:Z<l>", "fwd:Y", "fwd:Zu", "fwd:Zv" (GEMMs on the stored operand) and "gate:G<l>" /
    "mix:G<l>" (the kernels after each hidden layer)."""
    net, cr = plan.compiled.net, plan.compiled
    L = len(net.widths) - 1
    gp = gate_params(net)
    blocks = param_blocks(net.widths)
    e: Dict[str, float] = {}
    S, Sa = seeds(plan, views, params), seeds(plan, views, params, True)

    def operand(l):
        return (S, Sa) if l == 1 else (views[f"G{l - 1}"].double(), views[f"G{l - 1}"].double().abs())

    for l in range(1, L + 1):
        w_sl, b_sl, (K, N) = blocks[l - 1]
        A, Aa = operand(l)
        e[f"fwd:Z{l}" if l < L else "fwd:Y"] = layer_errors(
            cr, None, A, params[w_sl].view(K, N), params[b_sl], A_abs=Aa,
            out=views[f"Z{l}"] if l < L else views["Y"])["fwd"]
    A, Aa = operand(emb_of(net) + 1)
    for k, (ws, bs) in (("u", (gp.Wu, gp.bu)), ("v", (gp.Wv, gp.bv))):
        e[f"fwd:Z{k}"] = layer_errors(cr, None, A, params[ws].view(gp.K, gp.H), params[bs], A_abs=Aa,
                                      out=views[f"Z{k}"])["fwd"]
    Zu, Zv = views["Zu"].double(), views["Zv"].double()
    for l in range(1, L):
        Z = views[f"Z{l}"].double()
        kind = post_kind(net, l)
        if kind == "gate":
            ref, ra = gate_expr(net.act, Z, Zu, Zv, cr), gate_expr(net.act, Z, Zu, Zv, cr, absolute=True)
        else:
            a, Xp = (_alpha(net, params, l), views[f"G{l - 3}"].double()) if kind == "mix" else (None, None)
            ref, ra = mix_expr(act_of(net, l), Z, a, Xp, cr), mix_expr(act_of(net, l), Z, a, Xp, cr, absolute=True)
        e[f"{'gate' if kind == 'gate' else 'mix'}:G{l}"] = _cw_err(views[f"G{l}"], ref, ra)
    return e


def _alpha(net, params, l: int) -> torch.Tensor:
    """alpha of the block whose adaptive residual follows hidden layer l."""
    return params[gate_params(net).alpha][(l - 2) // 3].double()


def backward_errors(plan, views: Dict[str, torch.Tensor], params: torch.Tensor,
                    block: int = 8192) -> Tuple[Dict[str, float], torch.Tensor, torch.Tensor]:
    """Every adjoint pass from the engine's stored Zbar_{l+1} (the views of a PPSCI_B200_KEEP_ADJOINTS plan):
    "dx:Zbar<l>" for every hidden layer, "zub:u" / "zub:v" (Zubar / Zvbar summed over the gates) and "xres"
    (PirateNet); also the reference dLoss/d alpha per block and its componentwise bound (``alpha_errors``)."""
    net, cr = plan.compiled.net, plan.compiled
    L = len(net.widths) - 1
    gp = gate_params(net)
    blocks = param_blocks(net.widths)
    emb = emb_of(net)
    W = {l: params[blocks[l - 1][0]].view(*blocks[l - 1][2]).double() for l in range(2, L + 1)}
    Wu, Wv = (params[s].view(gp.K, gp.H).double() for s in (gp.Wu, gp.Wv))
    n = views["Z1"].shape[1]
    dx = {l: _PlaneMax() for l in range(1, L)}
    zub, zvb, xres = _PlaneMax(), _PlaneMax(), _PlaneMax()
    nb = n_blocks(net)
    da = torch.zeros(nb, dtype=torch.float64, device=params.device)
    da_abs = torch.zeros_like(da)
    for p0 in range(0, n, block):
        sl = slice(p0, min(n, p0 + block))
        v = {k: t[:, sl].double().clone() for k, t in views.items() if k != "X"}
        Zu = v["Zu"].requires_grad_(True)
        Zv = v["Zv"].requires_grad_(True)
        U_ref = torch.zeros_like(Zu)
        V_ref = torch.zeros_like(Zv)
        x_res = None  # carried residual adjoint (reference chain)
        for l in range(L - 1, 0, -1):
            zb_next = v[f"Zbar{l + 1}"] if l + 1 < L else v["Ybar"]
            gbar = zb_next @ W[l + 1].T
            gbar_abs = zb_next.abs() @ W[l + 1].abs().T
            if emb and l == 1:
                gbar = gbar + v["Zub"] @ Wu.T + v["Zvb"] @ Wv.T
            kind = post_kind(net, l)
            Z = v[f"Z{l}"].detach().requires_grad_(True)
            if kind == "gate":
                G = gate_expr(net.act, Z, Zu, Zv, cr)
                gz, gu, gv = torch.autograd.grad(G, (Z, Zu, Zv), grad_outputs=gbar)
                U_ref += gu
                V_ref += gv
            elif kind == "mix":
                b = (l - 2) // 3
                a = _alpha(net, params, l).detach().requires_grad_(True)
                Xp = v[f"G{l - 3}"].detach().requires_grad_(True)
                use_res = l != L - 1  # the last block's output feeds the output layer only
                xb = gbar + x_res if use_res else gbar
                xb_abs = gbar_abs + x_res.abs() if use_res else gbar_abs
                X = mix_expr(act_of(net, l), Z, a, Xp, cr)
                gz, ga, gx = torch.autograd.grad(X, (Z, a, Xp), grad_outputs=xb)
                x_res = gx
                da[b] += ga
                da_abs[b] += (xb_abs * (act_abs(act_of(net, l), Z.detach(), cr) + Xp.detach().abs())).sum()
                if l == 4:
                    xres.add(v["Xres"], x_res)
            else:  # embedding layer: X = act_first(Z), plus the residual path of block 0 (PirateNet)
                X = mix_expr(act_of(net, 1), Z, None, None, cr)
                xb = gbar + x_res if net.gated == 2 else gbar
                (gz,) = torch.autograd.grad(X, (Z,), grad_outputs=xb)
            dx[l].add(v[f"Zbar{l}"], gz)
        zub.add(v["Zub"], U_ref)
        zvb.add(v["Zvb"], V_ref)
    e = {f"dx:Zbar{l}": m.value() for l, m in dx.items()}
    e["zub:u"], e["zub:v"] = zub.value(), zvb.value()
    if net.gated == 2:
        e["xres"] = xres.value()
    return e, da, da_abs


def alpha_errors(plan, grads: torch.Tensor, da: torch.Tensor, da_abs: torch.Tensor,
                 seed: Optional[torch.Tensor] = None) -> Dict[str, float]:
    """"alpha:<b>": dLoss/d alpha of block b in ``grads`` (accumulated onto ``seed`` if given) against the reference
    of ``backward_errors``."""
    sl = gate_params(plan.compiled.net).alpha
    got = grads[sl].double()
    if seed is not None:
        s = seed[sl].double()
        got, da_abs = got - s, da_abs + s.abs()
    return {f"alpha:{b}": _cw_err(got[b: b + 1], da[b: b + 1], da_abs[b: b + 1]) for b in range(da.numel())}


def param_errors(plan, views: Dict[str, torch.Tensor], params: torch.Tensor, grads: torch.Tensor,
                 seed: Optional[torch.Tensor] = None) -> Dict[str, float]:
    """dW_l / db_l of every layer ("dw:W<l>", "db:b<l>"), of the embeddings ("dw:Wu", "db:bu", ...) and, with
    trainable frequencies, "omega", from the engine's Zbar_l (a PPSCI_B200_KEEP_ADJOINTS plan's views), accumulated
    onto ``seed`` if given."""
    net, cr = plan.compiled.net, plan.compiled
    L = len(net.widths) - 1
    gp = gate_params(net)
    blocks = param_blocks(net.widths)
    S, Sa = seeds(plan, views, params), seeds(plan, views, params, True)
    e: Dict[str, float] = {}

    def operand(l):
        return (S, Sa) if l == 1 else (views[f"G{l - 1}"].double(), views[f"G{l - 1}"].double().abs())

    def seeded(ws, bs, shape):
        return {"seed": (seed[ws].view(*shape), seed[bs])} if seed is not None else {}

    for l in range(1, L + 1):
        w_sl, b_sl, (K, N) = blocks[l - 1]
        A, Aa = operand(l)
        r = layer_errors(cr, None, A, params[w_sl].view(K, N), params[b_sl], A_abs=Aa,
                         zbar=views[f"Zbar{l}"] if l < L else views["Ybar"], dw=grads[w_sl].view(K, N),
                         db=grads[b_sl], **seeded(w_sl, b_sl, (K, N)))
        e[f"dw:W{l}"], e[f"db:b{l}"] = r["dw"], r["db"]
    A, Aa = operand(emb_of(net) + 1)
    for k, (ws, bs) in (("u", (gp.Wu, gp.bu)), ("v", (gp.Wv, gp.bv))):
        r = layer_errors(cr, None, A, params[ws].view(gp.K, gp.H), params[bs], A_abs=Aa, zbar=views[f"Z{k}b"],
                         dw=grads[ws].view(gp.K, gp.H), db=grads[bs], **seeded(ws, bs, (gp.K, gp.H)))
        e[f"dw:W{k}"], e[f"db:b{k}"] = r["dw"], r["db"]
    if net.n_omega:
        w_sl, _, (K, N) = blocks[0]
        cons = [(views["Zbar1"], params[w_sl].view(K, N))]
        if not emb_of(net):  # embed_u / embed_v read the seeds too
            cons += [(views["Zub"], params[gp.Wu].view(gp.K, gp.H)), (views["Zvb"], params[gp.Wv].view(gp.K, gp.H))]
        e["omega"] = omega_errors(plan, views, params, grads, seed=seed, consumers=cons)
    return e


# ------------------------------------------------------------------------------------------------------------------
# a gated case
# ------------------------------------------------------------------------------------------------------------------
@contextmanager
def _keep_env(keep: bool):
    old = os.environ.get(KEEP_ENV)
    if keep:
        os.environ[KEEP_ENV] = "1"
    else:
        os.environ.pop(KEEP_ENV, None)
    try:
        yield
    finally:
        if old is None:
            os.environ.pop(KEEP_ENV, None)
        else:
            os.environ[KEEP_ENV] = old


@dataclass
class GatedRun:
    cr: object
    dtype: torch.dtype
    params: torch.Tensor
    inputs: Dict[str, torch.Tensor]
    labels: Dict[str, torch.Tensor]
    n: int
    library: object


def setup(layout: str, gated: int, hidden: Sequence[int], n: int, *, dtype=torch.float32, act: str = "tanh",
          act_first: Optional[str] = None, alphas: Optional[Sequence[float]] = None,
          periods: Optional[Dict[str, Tuple[float, bool]]] = None, library=None, device="cuda:0",
          seed: int = 0) -> GatedRun:
    """A gated network on the layout's equation: ``gated`` 1 (ModifiedMLP; with ``act_first`` layer 1 is an
    embedding layer whose output feeds embed_u / embed_v) or 2 (PirateNet: layer 1 the embedding, then blocks of
    three layers), hidden widths ``hidden`` (layer 1 first), seeded random parameters with the blocks' ``alphas``.
    ``periods`` as in ``layer_ref.run_fused``."""
    spec = all_layouts()[layout]
    torch.manual_seed(seed)
    net = make_net(spec["in_keys"], spec["out_keys"], hidden, act, periods, gated=gated)
    net.act_first = act_first
    if periods and any(t for _, t in periods.values()):
        keys = [k for k, (_, t) in periods.items() if t]
        net.feat_omega_param = [keys.index(net.input_keys[s]) if (kind and net.input_keys[s] in keys) else -1
                                for s, kind in zip(net.feat_src, net.feat_kind)]
        net.n_omega = len(keys)
    cr = compile_residuals(net, spec["exprs"]())
    assert cr.channels == spec["C"], (layout, cr.channels)
    params = O.xavier_uniform_params(net.widths, 1, torch.float64)
    params = params + 0.1 * torch.randn_like(params)
    gp = gate_params(net)
    lim = math.sqrt(6.0 / (gp.K + gp.H))
    emb_w = [(torch.rand(gp.K * gp.H, dtype=torch.float64) * 2 - 1) * lim, 0.1 * torch.randn(gp.H, dtype=torch.float64)]
    emb_w += [(torch.rand(gp.K * gp.H, dtype=torch.float64) * 2 - 1) * lim, 0.1 * torch.randn(gp.H, dtype=torch.float64)]
    nb = n_blocks(net)
    al = torch.tensor(list(alphas) if alphas is not None else [0.3] * nb, dtype=torch.float64)
    assert al.numel() == nb, (alphas, nb)
    extra = [al]
    if net.n_omega:
        keys = [k for k, (_, t) in periods.items() if t]
        extra.append(torch.tensor([1.1 * 2 * math.pi / periods[k][0] for k in keys], dtype=torch.float64))
    params = torch.cat([params] + emb_w + extra).to(dtype)
    assert params.numel() == net.n_params and omega_offset(net) == params.numel() - net.n_omega
    inputs = {}
    for k in spec["in_keys"]:
        lo, hi = spec.get("ranges", {}).get(k, (0, 1))
        inputs[k] = (torch.rand(n, 1, dtype=torch.float64) * (hi - lo) + lo).to(dtype)
    labels = {k: (torch.randn(n, 1, dtype=torch.float64).to(dtype) if spec.get("labels_rand") else
                  torch.zeros(n, 1, dtype=dtype)) for k in cr.names}
    dev = torch.device(device)
    return GatedRun(cr, dtype, params.to(dev), {k: t.to(dev) for k, t in inputs.items()},
                    {k: t.to(dev) for k, t in labels.items()}, n, library)


def make_plan(run: GatedRun, keep: bool, chunk_points: int = 0) -> ResidualPlan:
    with _keep_env(keep):
        nres = len(run.cr.names)
        return ResidualPlan(run.cr, run.dtype, ["mean"] * nres, [1.0 + 0.5 * k for k in range(nres)], backend=1,
                            library=run.library, chunk_points=chunk_points)


def call(run: GatedRun, plan: ResidualPlan, grads0: Optional[torch.Tensor] = None, poison: Optional[int] = None):
    """One fused loss_fwd_bwd: (losses, grads, views of the last chunk with "X" the raw inputs of its points)."""
    ws = plan._workspace(run.n, run.params.device)
    if poison is not None:
        ws.fill_(poison)
    grads = grads0.clone() if grads0 is not None else torch.zeros_like(run.params)
    loss = plan.loss_fwd_bwd(run.inputs, run.params, grads, labels=run.labels).clone()
    last = run.n > plan.chunk_points
    keep = int(plan.lib.lib.ppsci_b200_plan_stash_offset(plan.handle, run.n, CODE_ZBAR_KEEP + 1)) >= 0
    views = gated_views(plan, run.n, last=last, keep=keep)
    x_off, n_last = last_chunk(plan, run.n) if last else (0, run.n)
    views["X"] = torch.stack([run.inputs[k].view(-1)[x_off: x_off + n_last] for k in run.cr.net.input_keys])
    return loss, grads, views


def grad_errors(plan, views, params, grads, da, da_abs, seed=None) -> Dict[str, float]:
    """``param_errors`` and ``alpha_errors`` of one gradient buffer."""
    return {**param_errors(plan, views, params, grads, seed), **alpha_errors(plan, grads, da, da_abs, seed)}


def _bitwise(a: torch.Tensor, b: torch.Tensor) -> bool:
    it = {1: torch.uint8, 4: torch.int32, 8: torch.int64}[a.element_size()]
    return a.shape == b.shape and a.dtype == b.dtype and bool(torch.equal(a.contiguous().view(it), b.contiguous().view(it)))


def _losses_agree(a: torch.Tensor, b: torch.Tensor, n: int, u: float) -> bool:
    """The head kernel's blocks add fp64 partial losses atomically, in any order: within the rounding of that sum."""
    blocks = (n + 127) // 128
    if blocks == 1:
        return _bitwise(a, b)
    return torch.allclose(a.double(), b.double(), rtol=(blocks + 4) * max(u, 2.0 ** -53), atol=0)


@dataclass(frozen=True)
class Case:
    layout: str
    gated: int
    hidden: Tuple[int, ...]
    n: int
    dtype: torch.dtype = torch.float32
    act: str = "tanh"
    act_first: Optional[str] = None
    alphas: Optional[Tuple[float, ...]] = None
    periods: Optional[Tuple[Tuple[str, float, bool], ...]] = None  # (input key, period, trainable)
    chunked: bool = False  # also a call over three workspace chunks
    seeded: bool = False  # also a call whose gradient buffer starts at G0

    @property
    def name(self) -> str:
        kind = {1: "mmlp" if self.act_first is None else f"mmlp_{self.act_first}", 2: "pirate"}[self.gated]
        s = f"{kind}-{self.layout}-h{'-'.join(map(str, self.hidden))}-n{self.n}-" \
            f"{'f64' if self.dtype == torch.float64 else 'f32'}-{self.act}"
        if self.alphas is not None:
            s += "-a" + "_".join(f"{a:g}" for a in self.alphas)
        if self.periods:
            s += "-p" + "".join(f"{k}{'T' if t else 'F'}" for k, _, t in self.periods)
        return s + ("-chunked" if self.chunked else "") + ("-seeded" if self.seeded else "")


GATE_PLANES = ("Y", "Ybar", "Zu", "Zv", "Zub", "Zvb", "Xres", "Zbar1", "Zbar2")


def run_case(case: Case, *, library=None, device="cuda:0") -> Dict[str, float]:
    """Every check of ``case``, raw relative errors keyed "<pass>:<plane>[@<call>]":
    * a PPSCI_B200_KEEP_ADJOINTS call on a zeroed workspace: every forward, adjoint and gradient pass;
    * a default call on a workspace of NaN bytes: Z_l, G_l, Y, Ybar, Zu, Zv, Zubar, Zvbar, Xres, Zbar_1 and Zbar_2 bitwise
      equal to the first call's, the losses within their summation order, and its gradient against the reference
      ("@default"; dW, d alpha and d omega are summed with atomics);
    * ``plan.forward``: Y bitwise equal;
    * ``seeded``: the gradient buffer seeded with G0, every block G0 + gradient ("@acc");
    * ``chunked``: a call over three workspace chunks, the forward and adjoint planes of the last one ("@chunk")."""
    periods = {k: (p, t) for k, p, t in case.periods} if case.periods else None
    run = setup(case.layout, case.gated, case.hidden, case.n, dtype=case.dtype, act=case.act, act_first=case.act_first,
                alphas=case.alphas, periods=periods, library=library, device=device)
    u = 2.0 ** -24 if case.dtype == torch.float32 else 2.0 ** -53
    n = case.n
    net = run.cr.net
    L = len(net.widths) - 1
    plan = make_plan(run, keep=True, chunk_points=n)
    assert plan.chunk_points >= n
    plan._workspace(n, run.params.device).zero_()
    loss, grads, V = call(run, plan)
    # the stash is not all zeros (a wrong offset into zeroed memory would pass the comparisons); with alpha = 0 in every
    # block no adjoint reaches the gates
    live = [k for k in ("Ybar", "Zub", "Zvb") if k == "Ybar" or case.gated == 1 or any(run.params[gate_params(net).alpha] != 0)]
    for k in live:
        assert float(V[k].abs().max()) > 0, f"{k} is all zeros"
    e = forward_errors(plan, V, run.params)
    eb, da, da_abs = backward_errors(plan, V, run.params)
    e.update(eb)
    e.update(grad_errors(plan, V, run.params, grads, da, da_abs))

    plan_d = make_plan(run, keep=False, chunk_points=n)
    loss_d, grads_d, Vd = call(run, plan_d, poison=0xFF)
    names = [f"Z{l}" for l in range(1, L)] + [f"G{l}" for l in range(1, L)] + [k for k in GATE_PLANES if k in Vd]
    for k in names:
        assert _bitwise(Vd[k], V[k]), f"default workspace layout on NaN bytes: {k} differs"
    assert _losses_agree(loss_d, loss, n, u), f"default workspace layout on NaN bytes: losses {loss_d} != {loss}"
    e.update({f"{k}@default": v for k, v in grad_errors(plan, V, run.params, grads_d, da, da_abs).items()})
    jets, _ = plan_d.forward(run.inputs, run.params, want_jets=True, want_residuals=False)
    assert _bitwise(jets, V["Y"].contiguous()), "plan.forward: Y differs"

    if case.seeded:
        gen = torch.Generator().manual_seed(7)
        g0 = (torch.randn(grads.numel(), generator=gen, dtype=torch.float64) * float(grads.double().std()))
        g0 = g0.to(case.dtype).to(run.params.device)
        _, grads_s, Vs = call(run, plan, grads0=g0)
        e.update({f"{k}@acc": v for k, v in grad_errors(plan, Vs, run.params, grads_s, da, da_abs, seed=g0).items()})

    if case.chunked:
        plan_c = make_plan(run, keep=True, chunk_points=-(-n // 3))
        _, _, Vc = call(run, plan_c)
        assert Vc["Z1"].shape[1] == n - 2 * plan_c.chunk_points
        ec = forward_errors(plan_c, Vc, run.params)
        ec.update(backward_errors(plan_c, Vc, run.params)[0])
        e.update({f"{k}@chunk": v for k, v in ec.items()})
    return e
