from __future__ import annotations

from typing import Union

from . import base


class HeatExchanger(base.PDE):
    r"""Heat exchanger equations (reference: ppsci/equation/pde/heat_exchanger.py:21-94): hot fluid, cold fluid and wall

    .. math::
        T_{h,t} + v_h T_{h,x} = \beta_h (T_w - T_h),\quad T_{c,t} - v_c T_{c,x} = \beta_c (T_w - T_c),\quad
        T_{w,t} = w_h (T_h - T_w) + w_c (T_c - T_w),\qquad \beta_h = \alpha_h v_h / q_{m,h},\ \beta_c = \alpha_c v_c / q_{m,c}

    over T_h(x, t, qm_h), T_c(x, t, qm_c) and T_w(x, t); the mass flow rates qm_h, qm_c are input columns.

    Args:
        alpha_h: (eta_o alpha A)_h / (L (c_p)_h)
        alpha_c: (eta_o alpha A)_c / (L (c_p)_c)
        v_h: flow velocity of the hot fluid
        v_c: flow velocity of the cold fluid
        w_h: (eta_o alpha A)_h / (M (c_p)_w)
        w_c: (eta_o alpha A)_c / (M (c_p)_w)
    """

    def __init__(
        self,
        alpha_h: Union[float, str],
        alpha_c: Union[float, str],
        v_h: Union[float, str],
        v_c: Union[float, str],
        w_h: Union[float, str],
        w_c: Union[float, str],
    ):
        super().__init__()
        x, t, qm_h, qm_c = self.create_symbols("x t qm_h qm_c")

        T_h = self.create_function("T_h", (x, t, qm_h))
        T_c = self.create_function("T_c", (x, t, qm_c))
        T_w = self.create_function("T_w", (x, t))

        beta_h = (alpha_h * v_h) / qm_h
        beta_c = (alpha_c * v_c) / qm_c

        self.add_equation("heat_boundary", T_h.diff(t) + v_h * T_h.diff(x) - beta_h * (T_w - T_h))
        self.add_equation("cold_boundary", T_c.diff(t) - v_c * T_c.diff(x) - beta_c * (T_w - T_c))
        self.add_equation("wall", T_w.diff(t) - w_h * (T_h - T_w) - w_c * (T_c - T_w))

        self._apply_detach()
