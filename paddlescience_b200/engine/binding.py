"""ctypes binding of the C-ABI declared in ``include/ppsci_b200.h``.

The product path loads ``paddlescience_b200/lib/libppsci_b200.so`` (hand-written sm_90a CUDA,
built in-tree by ``paddlescience_b200.engine.build``).  There is NO CPU fallback: if the
library is missing or no H100 is visible, every compute entry point raises.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

MAX_IN = 8
MAX_FEAT = 32
MAX_LAYERS = 16
MAX_DIR = 8
MAX_ORDER = 4
MAX_RES = 16
MAX_REG = 256
MAX_PGRAD = 32

F32, F64 = 0, 1

ACT_IDS = {
    "tanh": 0,
    "sin": 1,
    "cos": 2,
    "sigmoid": 3,
    "silu": 4,
    "swish": 4,
    "identity": 5,
    "relu": 6,
    "gelu": 7,
    "elu": 8,
    "selu": 9,
    "leaky_relu": 10,
    "siren": 11,
    # activations with a trainable parameter (plain MLP plans; their betas sit behind the other parameters)
    "stan": 12,     # tanh(x) (1 + beta x), one beta per unit
    "swish_b": 13,  # x sigmoid(beta x), one beta per layer: what arch.MLP(activation="swish") runs (the reference's Swish);
                    # plain "swish" above is the fixed-beta form (DeepONet sub-networks)
}

OPS = {
    "const": 0, "mov": 1, "add": 2, "sub": 3, "mul": 4, "div": 5, "neg": 6, "powi": 7, "pow": 8,
    "sin": 9, "cos": 10, "tanh": 11, "exp": 12, "log": 13, "sqrt": 14, "abs": 15, "max": 16,
    "min": 17, "sign": 18, "fma": 19, "sinh": 20, "cosh": 21, "heaviside": 22,
}

REDUCE_MEAN, REDUCE_SUM = 0, 1


class PlanSpec(C.Structure):
    """Mirror of ``ppsci_plan_spec`` (include/ppsci_b200.h)."""

    _fields_ = [
        ("dtype", C.c_int32),
        ("n_in", C.c_int32),
        ("n_feat", C.c_int32),
        ("feat_src", C.c_int32 * MAX_FEAT),
        ("feat_kind", C.c_int32 * MAX_FEAT),
        ("feat_omega", C.c_double * MAX_FEAT),
        ("n_layers", C.c_int32),
        ("widths", C.c_int32 * (MAX_LAYERS + 1)),
        ("act", C.c_int32),
        ("n_dir", C.c_int32),
        ("dir_order", C.c_int32 * MAX_DIR),
        ("dir_vec", (C.c_double * MAX_IN) * MAX_DIR),
        ("n_aux", C.c_int32),
        ("n_reg", C.c_int32),
        ("n_ops", C.c_int32),
        ("prog", C.POINTER(C.c_int32)),
        ("n_consts", C.c_int32),
        ("consts", C.POINTER(C.c_double)),
        ("n_res", C.c_int32),
        ("res_reg", C.c_int32 * MAX_RES),
        ("n_grad", C.c_int32),
        ("grad_res", C.POINTER(C.c_int32)),
        ("grad_in", C.POINTER(C.c_int32)),
        ("grad_reg", C.POINTER(C.c_int32)),
        ("reduction", C.c_int32 * MAX_RES),
        ("loss_weight", C.c_double * MAX_RES),
        ("chunk_points", C.c_int32),
        ("backend", C.c_int32),
        ("dense_in", C.c_int32),
        ("act_first", C.c_int32),
        ("aux_bcast", C.c_int32 * MAX_IN),
        ("n_pgrad", C.c_int32),
        ("pgrad_res", C.c_int32 * MAX_PGRAD),
        ("pgrad_aux", C.c_int32 * MAX_PGRAD),
        ("pgrad_reg", C.c_int32 * MAX_PGRAD),
        ("gated", C.c_int32),
    ]


EXPORTED_SYMBOLS = (
    "ppsci_b200_plan_create",
    "ppsci_b200_plan_destroy",
    "ppsci_b200_plan_param_count",
    "ppsci_b200_plan_set_aux_grad",
    "ppsci_b200_plan_channels",
    "ppsci_b200_plan_workspace_bytes",
    "ppsci_b200_residual_loss_fwd_bwd",
    "ppsci_b200_residual_fwd",
    "ppsci_b200_values_fwd_bwd",
    "ppsci_b200_values_fwd_keep",
    "ppsci_b200_values_bwd_kept",
    "ppsci_b200_plan_chunk_points",
    "ppsci_b200_deeponet_head",
    "ppsci_b200_sample_uniform",
    "ppsci_b200_plan_last_launches",
    "ppsci_b200_plan_uses_tcgen05",
    "ppsci_b200_plan_stash_offset",
    "ppsci_b200_plan_set_profile",
    "ppsci_b200_plan_get_profile",
    "ppsci_b200_adam_step",
    "ppsci_b200_adam_step_dev",
    "ppsci_b200_last_error",
    "ppsci_b200_version",
)


def default_library_path() -> str:
    here = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    return os.path.join(here, "lib", "libppsci_b200.so")


class EngineError(RuntimeError):
    pass


class Library:
    """A loaded C-ABI library with typed entry points."""

    def __init__(self, path: Optional[str] = None):
        self.path = path or default_library_path()
        if not os.path.exists(self.path):
            raise EngineError(
                f"native library not found at {self.path}; build it with "
                "`python -c 'import __graft_entry__ as g; g.build()'` "
                "(the engine has no CPU fallback)"
            )
        self.lib = C.CDLL(self.path)
        L = self.lib
        vp, i64, i32, dbl = C.c_void_p, C.c_int64, C.c_int32, C.c_double
        L.ppsci_b200_plan_create.argtypes = [C.POINTER(PlanSpec), C.POINTER(vp)]
        L.ppsci_b200_plan_create.restype = C.c_int
        L.ppsci_b200_plan_destroy.argtypes = [vp]
        L.ppsci_b200_plan_destroy.restype = None
        L.ppsci_b200_plan_param_count.argtypes = [vp]
        L.ppsci_b200_plan_param_count.restype = i64
        L.ppsci_b200_plan_set_aux_grad.argtypes = [vp, C.c_int32, vp]
        L.ppsci_b200_plan_set_aux_grad.restype = C.c_int
        L.ppsci_b200_plan_channels.argtypes = [vp]
        L.ppsci_b200_plan_channels.restype = i32
        L.ppsci_b200_plan_workspace_bytes.argtypes = [vp, i64]
        L.ppsci_b200_plan_workspace_bytes.restype = C.c_size_t
        L.ppsci_b200_residual_loss_fwd_bwd.argtypes = [
            vp, C.POINTER(vp), C.POINTER(vp), C.POINTER(vp), C.POINTER(dbl), C.POINTER(vp),
            i64, i64, vp, vp, vp, C.POINTER(vp), vp, C.c_size_t, vp,
        ]
        L.ppsci_b200_residual_loss_fwd_bwd.restype = C.c_int
        L.ppsci_b200_residual_fwd.argtypes = [
            vp, C.POINTER(vp), C.POINTER(vp), i64, vp, vp, C.POINTER(vp), vp, C.c_size_t, vp,
        ]
        L.ppsci_b200_residual_fwd.restype = C.c_int
        L.ppsci_b200_values_fwd_bwd.argtypes = [vp, C.POINTER(vp), C.POINTER(vp), i64, vp, vp, vp, vp, C.c_size_t, vp]
        L.ppsci_b200_values_fwd_bwd.restype = C.c_int
        L.ppsci_b200_values_fwd_keep.argtypes = [vp, C.POINTER(vp), C.POINTER(vp), i64, vp, vp, vp, C.c_size_t, vp]
        L.ppsci_b200_values_fwd_keep.restype = C.c_int
        L.ppsci_b200_values_bwd_kept.argtypes = [vp, C.POINTER(vp), C.POINTER(vp), i64, vp, vp, vp, vp, C.c_size_t, vp]
        L.ppsci_b200_values_bwd_kept.restype = C.c_int
        L.ppsci_b200_plan_chunk_points.argtypes = [vp]
        L.ppsci_b200_plan_chunk_points.restype = i32
        L.ppsci_b200_deeponet_head.argtypes = [i32, i32, vp, vp, vp, vp, vp, i64, i32, dbl, vp, vp, vp, vp, vp, vp]
        L.ppsci_b200_deeponet_head.restype = C.c_int
        L.ppsci_b200_sample_uniform.argtypes = [i32, C.c_uint64, C.c_uint64, i64, i32, C.POINTER(dbl), C.POINTER(dbl), C.POINTER(vp), vp]
        L.ppsci_b200_sample_uniform.restype = C.c_int
        L.ppsci_b200_plan_last_launches.argtypes = [vp]
        L.ppsci_b200_plan_last_launches.restype = i64
        L.ppsci_b200_plan_uses_tcgen05.argtypes = [vp]
        L.ppsci_b200_plan_uses_tcgen05.restype = i32
        L.ppsci_b200_plan_stash_offset.argtypes = [vp, i64, i32]
        L.ppsci_b200_plan_stash_offset.restype = i64
        L.ppsci_b200_plan_set_profile.argtypes = [vp, i32]
        L.ppsci_b200_plan_set_profile.restype = C.c_int
        L.ppsci_b200_plan_get_profile.argtypes = [vp, C.POINTER(dbl), C.POINTER(i64)]
        L.ppsci_b200_plan_get_profile.restype = C.c_int
        L.ppsci_b200_adam_step.argtypes = [i32, vp, vp, vp, vp, i64, dbl, dbl, dbl, dbl, dbl, i64, dbl, vp]
        L.ppsci_b200_adam_step.restype = C.c_int
        L.ppsci_b200_adam_step_dev.argtypes = [i32, vp, vp, vp, vp, i64, vp, dbl, dbl, dbl, dbl, i32, vp]
        L.ppsci_b200_adam_step_dev.restype = C.c_int
        L.ppsci_b200_last_error.argtypes = []
        L.ppsci_b200_last_error.restype = C.c_char_p
        L.ppsci_b200_version.argtypes = []
        L.ppsci_b200_version.restype = C.c_char_p

    def last_error(self) -> str:
        return self.lib.ppsci_b200_last_error().decode()

    def version(self) -> str:
        return self.lib.ppsci_b200_version().decode()

    def check(self, rc: int, what: str) -> None:
        if rc != 0:
            raise EngineError(f"{what}: {self.last_error()}")


_default: Optional[Library] = None


def get_library() -> Library:
    """The product library (CUDA).  Raises EngineError when it is not built."""
    global _default
    if _default is None:
        _default = Library()
    return _default
