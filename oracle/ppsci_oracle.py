"""CPU ORACLE — TEST INFRASTRUCTURE ONLY.  Never imported by ``paddlescience_b200``.

A plain PyTorch (CPU, autograd) restatement of the reference's hot path, following the
reference's own algorithm: reverse-mode ``grad(create_graph=True)`` sweeps per derivative
order, node-by-node evaluation of the sympy residual, MSE, and ``backward()`` to the weights.
Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s cpu_baseline / ``--impl reference``
leg may import this module, and only as the checker / the timed CPU baseline.

PARITY PINNING STATUS: "parity unpinned" against PaddlePaddle's absolute outputs — the
arithmetic of the reference lives in the third-party ``paddlepaddle`` package, which is neither
vendored in /root/reference nor installable here (no wheel, no network; every ``ppsci`` module
imports it at top level), and the reference's tests hold no absolute golden vectors for this
path (SURVEY.md §8c).  What IS pinned, and checked in tests/test_oracle.py:
  * ``MSELoss`` docstring known answers (ppsci/loss/mse.py:51-68)
  * the reference's own relative test designs (test/equation/test_navier_stokes.py:80-178,
    test_laplace.py, test_biharmonic.py, test_detach.py, test/utils/test_symbolic.py:93-149):
    equation-via-expression == hand-written jacobian/hessian on the same network
  * geometry sampling docstring arrays (ppsci/geometry/geometry.py:157-183)
  * fp64 vs fp32 self-consistency (fp64 run is treated as ground truth).

Each function cites the reference file:line it restates.
"""
from __future__ import annotations

import math
from typing import Callable, Dict, List, Optional, Sequence, Tuple, Union

import numpy as np
import sympy as sp
import torch
from sympy.core.function import AppliedUndef

DETACH_FUNC_NAME = "detach"  # ppsci/equation/pde/base.py:28


# ------------------------------------------------------------------------------------------------
# ppsci/arch/activation.py:139-154
# ------------------------------------------------------------------------------------------------
def get_activation(name: str) -> Callable[[torch.Tensor], torch.Tensor]:
    name = name.lower()
    table = {
        "tanh": torch.tanh,
        "sin": torch.sin,
        "cos": torch.cos,
        "sigmoid": torch.sigmoid,
        "silu": lambda x: x * torch.sigmoid(x),  # activation.py:71-83 (x*sigmoid(x) workaround)
        "swish": lambda x: x * torch.sigmoid(x),  # activation.py:45-55 with beta = 1
        "identity": lambda x: x,
        "relu": torch.relu,
        "gelu": lambda x: torch.nn.functional.gelu(x),
        # paddle defaults (activation.py:139-145): nn.ELU(alpha=1.0), nn.SELU(), nn.LeakyReLU(negative_slope=0.01)
        "elu": lambda x: torch.where(x > 0, x, torch.exp(x) - 1),
        "selu": lambda x: 1.0507009873554804934193349852946 * torch.where(x > 0, x, 1.6732632423543772848170429916717 * (torch.exp(x) - 1)),
        "leaky_relu": lambda x: torch.where(x > 0, x, 0.01 * x),
        "siren": lambda x: torch.sin(30.0 * x),  # Siren(w0=30).forward, activation.py:99-101
    }
    if name not in table:
        raise ValueError(f"act_name({name}) not found in act_func_dict")
    return table[name]


# ------------------------------------------------------------------------------------------------
# ppsci/arch/mlp.py:179-315 (+ base.py:78-148 concat/split, mlp.py:95-114 PeriodEmbedding)
# ------------------------------------------------------------------------------------------------
class OracleMLP:
    """Functional MLP over a flat parameter vector laid out as [W_1 (in,out), b_1, W_2, b_2, ...]
    (the reference's nn.Linear weight layout is [in, out], mlp.py:246,274)."""

    def __init__(
        self,
        input_keys: Sequence[str],
        output_keys: Sequence[str],
        hidden: Sequence[int],
        activation: str = "tanh",
        periods: Optional[Dict[str, Tuple[float, bool]]] = None,
        skip_connection: bool = False,
        fourier: Optional[Dict[str, float]] = None,
        modified: bool = False,
        pirate: bool = False,
        trainable_act: bool = False,
    ):
        # trainable_act=True with activation "stan" / "swish": the reference's activation LAYERS carry parameters —
        # Stan.beta [hidden_i] (activation.py:28-46: tanh(x) (1 + beta x)) and Swish.beta [] (activation.py:49-58:
        # x sigmoid(beta x)), one layer instance per hidden layer (mlp.py:249-253, activation.py:169-171).  They are stored
        # behind the linear layers (and embeddings / alphas), hidden layer by hidden layer, in front of the fourier kernel.
        self.trainable_act = activation if (trainable_act and activation in ("stan", "swish")) else None
        if activation == "stan" and not trainable_act:
            raise ValueError("stan needs trainable_act=True (its beta is a parameter)")
        # pirate=True: PirateNet (mlp.py:530-830) — ``hidden`` holds one entry per block (all equal to the input width of
        # the blocks, i.e. fourier["dim"]); flat vector:
        # [block_0.linear1 | linear2 | linear3 | block_1... | last_fc | Wu | bu | Wv | bv | alpha_0..alpha_{B-1} | fourier kernel]
        self.pirate = pirate
        if pirate:
            self.n_blocks = len(hidden)
            hidden = [h for h in hidden for _ in range(3)]
        # modified=True: ModifiedMLP (mlp.py:318-506) — embed_u / embed_v (n_feat -> hidden[0]) stored BEHIND the linear
        # layers in the flat vector: [W_1 | b_1 | ... | W_L | b_L | Wu | bu | Wv | bv]
        self.modified = modified
        self.input_keys = tuple(input_keys)
        self.output_keys = tuple(output_keys)
        self.periods = periods or {}
        self.skip_connection = skip_connection
        n_feat = len(self.input_keys) + len(self.periods)  # mlp.py:222-226
        self.n_feat = n_feat
        # FourierEmbedding (mlp.py:117-136, 228-232): kernel [cur_size, dim // 2], then cur_size = dim.
        # Its kernel is stored BEHIND the linear layers in the flat vector: [W_1 | b_1 | ... | kernel].
        self.fourier = dict(fourier) if fourier else None
        first = int(self.fourier["dim"]) if self.fourier else n_feat
        self.widths = [first] + list(hidden) + [len(self.output_keys)]
        self.act = get_activation(activation) if activation != "stan" else None
        self.beta_len = ([int(h) for h in hidden] if self.trainable_act == "stan" else [1] * len(hidden)) if self.trainable_act else []

    @property
    def n_linear_params(self) -> int:
        return sum(a * b + b for a, b in zip(self.widths[:-1], self.widths[1:]))

    @property
    def n_params(self) -> int:
        n = self.n_linear_params + (self.n_feat * (int(self.fourier["dim"]) // 2) if self.fourier else 0)
        if self.modified or self.pirate:
            n += 2 * (self.widths[0] * self.widths[1] + self.widths[1])
        if self.pirate:
            n += self.n_blocks
        n += sum(self.beta_len)
        return n

    def split_params(self, flat: torch.Tensor):
        out, off = [], 0
        for a, b in zip(self.widths[:-1], self.widths[1:]):
            W = flat[off : off + a * b].view(a, b)
            off += a * b
            bias = flat[off : off + b]
            off += b
            out.append((W, bias))
        return out

    def __call__(self, flat: torch.Tensor, x: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        feats = []
        for k in self.input_keys:  # mlp.py:108-114 then base.py:109-112
            if k in self.periods:
                w = 2 * math.pi / float(self.periods[k][0])
                feats.append(torch.cat([torch.cos(w * x[k]), torch.sin(w * x[k])], dim=-1))
            else:
                feats.append(x[k])
        y = torch.cat(feats, dim=-1) if len(feats) > 1 else feats[0]
        if self.fourier:  # FourierEmbedding.forward, mlp.py:128-136; applied after the concat, mlp.py:306-309
            dh = int(self.fourier["dim"]) // 2
            koff = self.n_params - self.n_feat * dh  # the kernel is the LAST segment of the flat vector
            kernel = flat[koff : koff + self.n_feat * dh].view(self.n_feat, dh)
            y = torch.cat([torch.cos(y @ kernel), torch.sin(y @ kernel)], dim=-1)
        layers = self.split_params(flat)
        if self.pirate:  # PirateNet.forward_tensor (mlp.py:800-809) over PirateNetBlock.forward (mlp.py:617-624)
            a, h = self.widths[0], self.widths[1]
            off = self.n_linear_params
            Wu, bu = flat[off : off + a * h].view(a, h), flat[off + a * h : off + a * h + h]
            off += a * h + h
            Wv, bv = flat[off : off + a * h].view(a, h), flat[off + a * h : off + a * h + h]
            off += a * h + h
            alpha = flat[off : off + self.n_blocks]
            u = self.act(y @ Wu + bu)
            v = self.act(y @ Wv + bv)
            for k in range(self.n_blocks):
                (W1, b1), (W2, b2), (W3, b3) = layers[3 * k : 3 * k + 3]
                f = self.act(y @ W1 + b1)
                z1 = f * u + (1 - f) * v
                g = self.act(z1 @ W2 + b2)
                z2 = g * u + (1 - g) * v
                hh = self.act(z2 @ W3 + b3)
                y = alpha[k] * hh + (1 - alpha[k]) * y
            W, b = layers[-1]
            y = y @ W + b
            if len(self.output_keys) == 1:
                return {self.output_keys[0]: y}
            parts = torch.split(y, 1, dim=-1)
            return {k: parts[i] for i, k in enumerate(self.output_keys)}
        if self.modified:  # ModifiedMLP.forward_tensor, mlp.py:488-506
            a, h = self.widths[0], self.widths[1]
            off = self.n_linear_params
            Wu, bu = flat[off : off + a * h].view(a, h), flat[off + a * h : off + a * h + h]
            off += a * h + h
            Wv, bv = flat[off : off + a * h].view(a, h), flat[off + a * h : off + a * h + h]
            u = self.act(y @ Wu + bu)  # embed_u = Sequential(Linear, act), mlp.py:397-418
            v = self.act(y @ Wv + bv)
            skip = None
            for i, (W, b) in enumerate(layers[:-1]):  # mlp.py:494-504, statement by statement
                y = y @ W + b
                y = self.act(y)
                y = y * u + (1 - y) * v
                if self.skip_connection and i % 2 == 0:
                    if skip is not None:
                        skip = y
                        y = y + skip
                    else:
                        skip = y
            W, b = layers[-1]
            y = y @ W + b
            if len(self.output_keys) == 1:
                return {self.output_keys[0]: y}
            parts = torch.split(y, 1, dim=-1)
            return {k: parts[i] for i, k in enumerate(self.output_keys)}
        skip = None
        boff = self.n_params - sum(self.beta_len) - (self.n_feat * (int(self.fourier["dim"]) // 2) if self.fourier else 0)
        for i, (W, b) in enumerate(layers[:-1]):  # mlp.py:281-296, statement by statement
            y = y @ W + b
            if self.skip_connection and i % 2 == 0:
                if skip is not None:
                    skip = y
                    y = y + skip
                else:
                    skip = y
            if self.trainable_act == "stan":  # Stan.forward, activation.py:43-46
                beta = flat[boff : boff + self.beta_len[i]]
                boff += self.beta_len[i]
                y = torch.tanh(y) * (1 + beta * y)
            elif self.trainable_act == "swish":  # Swish.forward, activation.py:57-58
                beta = flat[boff]
                boff += 1
                y = y * torch.sigmoid(beta * y)
            else:
                y = self.act(y)
        W, b = layers[-1]
        y = y @ W + b
        if len(self.output_keys) == 1:
            return {self.output_keys[0]: y}
        parts = torch.split(y, 1, dim=-1)  # base.py:145-148
        return {k: parts[i] for i, k in enumerate(self.output_keys)}


def xavier_uniform_params(widths: Sequence[int], seed: int, dtype=torch.float64) -> torch.Tensor:
    """Flat parameters: Xavier-uniform weights, zero bias (Paddle nn.Linear default; SURVEY §7.1)."""
    g = torch.Generator().manual_seed(seed)
    chunks = []
    for a, b in zip(widths[:-1], widths[1:]):
        lim = math.sqrt(6.0 / (a + b))
        chunks.append(((torch.rand(a * b, generator=g, dtype=torch.float64) * 2 - 1) * lim).to(dtype))
        chunks.append(torch.zeros(b, dtype=dtype))
    return torch.cat(chunks)


# ------------------------------------------------------------------------------------------------
# ppsci/autodiff/ad.py:56-160 (jacobian), 196-303 (hessian)
# ------------------------------------------------------------------------------------------------
def jacobian(y: torch.Tensor, x: torch.Tensor) -> torch.Tensor:
    """d y / d x for y:[N,1], x:[N,1] by one reverse sweep, graph kept for higher orders
    (ad.py:73-75: paddle.grad(ys, xs, create_graph=True))."""
    (g,) = torch.autograd.grad(y, x, torch.ones_like(y), create_graph=True, allow_unused=True)
    if g is None:
        g = torch.zeros_like(x)
    return g


def hessian(y: torch.Tensor, x: torch.Tensor) -> torch.Tensor:
    """ad.py:196-236: jacobian of the (cached) jacobian."""
    return jacobian(jacobian(y, x), x)


# ------------------------------------------------------------------------------------------------
# ppsci/utils/symbolic.py:184-504 — node-by-node evaluation of a sympy residual
# ------------------------------------------------------------------------------------------------
def eval_expr(expr: sp.Basic, data: Dict[str, torch.Tensor]) -> torch.Tensor:
    """Evaluate ``expr`` over ``data`` (inputs with requires_grad, outputs attached to them).
    Derivative nodes follow DerivativeNode._derivate_operator_func (symbolic.py:310-333):
    successive first-order reverse sweeps in the order the variables are listed."""
    some = next(iter(data.values()))

    def ev(e: sp.Basic) -> torch.Tensor:
        if isinstance(e, sp.Derivative):
            f = e.args[0]
            if isinstance(f, AppliedUndef) and f.func.__name__ == DETACH_FUNC_NAME:
                f = f.args[0]  # base.py:138-148: detach on the first arg of Derivative is removed
            val = ev(f)
            for sym, order in e.variable_count:
                for _ in range(int(order)):
                    val = jacobian(val, data[str(sym)])
            return val
        if isinstance(e, AppliedUndef):
            nm = e.func.__name__
            if nm == DETACH_FUNC_NAME:
                return ev(e.args[0]).detach()  # DetachNode, symbolic.py:165-181
            return data[nm]
        if isinstance(e, sp.Symbol):
            return data[str(e)]
        if e.is_Number or isinstance(e, sp.NumberSymbol):
            return torch.full_like(some, float(e))
        if isinstance(e, sp.Add):
            acc = ev(e.args[0])
            for a in e.args[1:]:
                acc = acc + ev(a)
            return acc
        if isinstance(e, sp.Mul):
            acc = ev(e.args[0])
            for a in e.args[1:]:
                acc = acc * ev(a)
            return acc
        if isinstance(e, sp.Pow):
            base, ex = e.args
            if ex.is_Number:
                return torch.pow(ev(base), float(ex))
            return torch.pow(ev(base), ev(ex))
        table = {sp.sin: torch.sin, sp.cos: torch.cos, sp.tanh: torch.tanh, sp.exp: torch.exp, sp.log: torch.log,
                 sp.Abs: torch.abs, sp.sign: torch.sign, sp.sinh: torch.sinh, sp.cosh: torch.cosh, sp.tan: torch.tan}
        for cls, fn in table.items():
            if isinstance(e, cls):
                return fn(ev(e.args[0]))
        if isinstance(e, sp.Heaviside):  # a step: zero gradient, as paddle.heaviside
            a = ev(e.args[0]).detach()
            return torch.heaviside(a, torch.full_like(a, float(e.args[1]) if len(e.args) > 1 else 0.5))
        if isinstance(e, sp.Max):
            acc = ev(e.args[0])
            for a in e.args[1:]:
                acc = torch.maximum(acc, ev(a))
            return acc
        if isinstance(e, sp.Min):
            acc = ev(e.args[0])
            for a in e.args[1:]:
                acc = torch.minimum(acc, ev(a))
            return acc
        raise NotImplementedError(f"The node {e} is not supported in the oracle.")

    return ev(sp.sympify(expr))


# ------------------------------------------------------------------------------------------------
# ppsci/loss/mse.py:82-106
# ------------------------------------------------------------------------------------------------
def mse_loss(
    output_dict: Dict[str, torch.Tensor],
    label_dict: Dict[str, torch.Tensor],
    weight_dict: Optional[Dict[str, torch.Tensor]] = None,
    reduction: str = "mean",
    weight: Optional[Union[float, Dict[str, float]]] = None,
) -> Dict[str, torch.Tensor]:
    if reduction not in ("mean", "sum"):
        raise ValueError(f"reduction should be 'mean' or 'sum', but got {reduction}")
    losses = {}
    for key in label_dict:
        loss = (output_dict[key] - label_dict[key]) ** 2
        if weight_dict and key in weight_dict:
            loss = loss * weight_dict[key]
        if "area" in output_dict:
            loss = loss * output_dict["area"]
        loss = loss.sum() if reduction == "sum" else loss.mean()
        if isinstance(weight, (float, int)):
            loss = loss * weight
        elif isinstance(weight, dict) and key in weight:
            loss = loss * weight[key]
        losses[key] = loss
    return losses


# ------------------------------------------------------------------------------------------------
# ppsci/utils/expression.py:60-131 + ppsci/loss/mtl/sum.py:45-60 + ppsci/solver/train.py:158
# ------------------------------------------------------------------------------------------------
def train_forward_backward(
    model: OracleMLP,
    flat_params: torch.Tensor,
    exprs: Dict[str, Union[sp.Basic, Callable]],
    inputs: Dict[str, torch.Tensor],
    labels: Dict[str, torch.Tensor],
    weights: Optional[Dict[str, torch.Tensor]] = None,
    reduction: str = "mean",
    loss_weight: Optional[Union[float, Dict[str, float]]] = None,
    want_grad: bool = True,
):
    """One constraint of ExpressionSolver.train_forward followed by total_loss.backward().
    Returns (losses: {name: float tensor}, residuals: {name: [N,1]}, grad: flat tensor or None)."""
    params = flat_params.detach().clone().requires_grad_(want_grad)
    x = {k: v.detach().clone().requires_grad_(True) for k, v in inputs.items()}  # train.py:98-100
    out = model(params, {k: x[k] for k in model.input_keys})  # expression.py:96
    data = dict(x)
    data.update(out)
    residuals = {}
    for name, e in exprs.items():  # expression.py:101-102
        residuals[name] = e(data) if callable(e) and not isinstance(e, sp.Basic) else eval_expr(e, data)
    out_all = dict(out)
    out_all.update(residuals)
    losses = mse_loss(out_all, labels, weights, reduction, loss_weight)  # expression.py:112-116
    total = sum(losses.values())  # mtl/sum.py:45-60
    grad = None
    if want_grad:
        (grad,) = torch.autograd.grad(total, params, allow_unused=True)  # train.py:158
        if grad is None:
            grad = torch.zeros_like(params)
    return ({k: v.detach() for k, v in losses.items()}, {k: v.detach() for k, v in residuals.items()}, grad)


# ------------------------------------------------------------------------------------------------
# Equations, restated literally from ppsci/equation/pde/*.py (sympy construction only)
# ------------------------------------------------------------------------------------------------
def laplace_expr(dim: int) -> Dict[str, sp.Basic]:
    """ppsci/equation/pde/laplace.py:40-55"""
    invars = sp.symbols("x y z")[:dim]
    u = sp.Function("u")(*invars)
    e = 0
    for v in invars:
        e += u.diff(v, 2)
    return {"laplace": e}


def poisson_expr(dim: int) -> Dict[str, sp.Basic]:
    """ppsci/equation/pde/poisson.py:40-55"""
    invars = sp.symbols("x y z")[:dim]
    p = sp.Function("p")(*invars)
    e = 0
    for v in invars:
        e += p.diff(v, 2)
    return {"poisson": e}


def navier_stokes_expr(nu: float, rho: float, dim: int, time: bool) -> Dict[str, sp.Basic]:
    """ppsci/equation/pde/navier_stokes.py:70-151"""
    t, x, y, z = sp.symbols("t x y z")
    invars = (x, y)
    if time:
        invars = (t,) + invars
    if dim == 3:
        invars += (z,)
    u = sp.Function("u")(*invars)
    v = sp.Function("v")(*invars)
    w = sp.Function("w")(*invars) if dim == 3 else sp.Number(0)
    p = sp.Function("p")(*invars)
    eqs = {}
    eqs["continuity"] = u.diff(x) + v.diff(y) + w.diff(z)
    eqs["momentum_x"] = (u.diff(t) + u * u.diff(x) + v * u.diff(y) + w * u.diff(z)
                         - ((nu * u.diff(x)).diff(x) + (nu * u.diff(y)).diff(y) + (nu * u.diff(z)).diff(z))
                         + 1 / rho * p.diff(x))
    eqs["momentum_y"] = (v.diff(t) + u * v.diff(x) + v * v.diff(y) + w * v.diff(z)
                         - ((nu * v.diff(x)).diff(x) + (nu * v.diff(y)).diff(y) + (nu * v.diff(z)).diff(z))
                         + 1 / rho * p.diff(y))
    if dim == 3:
        eqs["momentum_z"] = (w.diff(t) + u * w.diff(x) + v * w.diff(y) + w * w.diff(z)
                             - ((nu * w.diff(x)).diff(x) + (nu * w.diff(y)).diff(y) + (nu * w.diff(z)).diff(z))
                             + 1 / rho * p.diff(z))
    return eqs


def biharmonic_expr(dim: int, q, D) -> Dict[str, sp.Basic]:
    """ppsci/equation/pde/biharmonic.py:45-74"""
    invars = sp.symbols("x y z")[:dim]
    u = sp.Function("u")(*invars)
    e = -sp.sympify(q) / sp.sympify(D)
    for vi in invars:
        for vj in invars:
            e += u.diff(vi, 2).diff(vj, 2)
    return {"biharmonic": e}


def allen_cahn_callable(eps: float) -> Dict[str, Callable]:
    """ppsci/equation/pde/allen_cahn.py:56-64 (a Python closure over jacobian)."""

    def allen_cahn(out):
        t, x = out["t"], out["x"]
        u = out["u"]
        u__t = jacobian(u, t)
        u__x = jacobian(u, x)
        u__x__x = jacobian(u__x, x)
        return u__t - (eps**2) * u__x__x + 5 * u * u * u - 5 * u

    return {"allen_cahn": allen_cahn}


# ------------------------------------------------------------------------------------------------
# Geometry sampling — ppsci/geometry/geometry_nd.py:83-115, sampler.py:49-57
# ------------------------------------------------------------------------------------------------
def hypercube_uniform_points(xmin, xmax, n: int, boundary: bool = True) -> np.ndarray:
    """geometry_nd.py:83-110 (float32 arithmetic, x slowest via itertools.product)."""
    import itertools

    xmin = np.array(xmin, dtype="float32")
    xmax = np.array(xmax, dtype="float32")
    side = xmax - xmin
    volume = np.prod(side, dtype="float32")
    ndim = len(xmin)
    dx = (volume / n) ** (1 / ndim)
    xi = []
    for i in range(ndim):
        ni = int(np.ceil(side[i] / dx))
        if boundary:
            xi.append(np.linspace(xmin[i], xmax[i], num=ni, dtype="float32"))
        else:
            xi.append(np.linspace(xmin[i], xmax[i], num=ni + 1, endpoint=False, dtype="float32")[1:])
    x = np.array(list(itertools.product(*xi)), dtype="float32")
    if len(x) > n:
        x = x[0:n]
    return x


def hypercube_random_points(xmin, xmax, n: int) -> np.ndarray:
    """geometry_nd.py:112-115 with sampler.pseudorandom (sampler.py:49-57)."""
    xmin = np.array(xmin, dtype="float32")
    xmax = np.array(xmax, dtype="float32")
    x = np.random.random(size=(n, len(xmin))).astype("float32")
    return (xmax - xmin) * x + xmin


# ------------------------------------------------------------------------------------------------
# ppsci/arch/deeponet.py:91-154  DeepONet:  G = einsum("bi,bi->b", branch(u), act(trunk(y))) [+ b]
# ------------------------------------------------------------------------------------------------
class OracleDeepONet:
    """Functional DeepONet over flat parameter vectors of its two MLPs (each laid out like OracleMLP) and the scalar
    bias.  branch: MLP((u,), ("b",), ..., input_dim=num_loc, output_dim=num_features) on the [N, num_loc] matrix
    (deeponet.py:96-106); trunk: MLP((y,), ("t",), ..., input_dim=1, output_dim=num_features) followed by the trunk
    activation (deeponet.py:108-119, 141-142); output reshaped to [N, 1] plus b (deeponet.py:144-149)."""

    def __init__(self, num_loc: int, num_features: int, branch_hidden: Sequence[int], trunk_hidden: Sequence[int],
                 branch_activation: str = "tanh", trunk_activation: str = "tanh", use_bias: bool = True):
        self.bw = [num_loc] + list(branch_hidden) + [num_features]
        self.tw = [1] + list(trunk_hidden) + [num_features]
        self.bact, self.tact = get_activation(branch_activation), get_activation(trunk_activation)
        self.use_bias = use_bias

    @staticmethod
    def _mlp(flat: torch.Tensor, widths: Sequence[int], act, x: torch.Tensor) -> torch.Tensor:
        off, y = 0, x
        n = len(widths) - 1
        for i, (a, b) in enumerate(zip(widths[:-1], widths[1:])):
            W = flat[off: off + a * b].view(a, b)
            off += a * b
            bias = flat[off: off + b]
            off += b
            y = y @ W + bias  # nn.Linear with [in, out] weights (mlp.py:246,274)
            if i < n - 1:
                y = act(y)  # mlp.py:281-296: activation after every hidden layer, none after last_fc
        return y

    def __call__(self, branch_params, trunk_params, b, u: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
        u_features = self._mlp(branch_params, self.bw, self.bact, u)
        y_features = self.tact(self._mlp(trunk_params, self.tw, self.tact, y))
        g = (u_features * y_features).sum(dim=-1).reshape(-1, 1)
        return g + b if self.use_bias else g
