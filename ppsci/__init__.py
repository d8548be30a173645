"""Import shim: ``import ppsci`` resolves to the H100-native implementation so that scripts
written against PaddleScience's hot-path API run unchanged (see INTEGRATION.md)."""
import sys as _sys

import paddlescience_b200 as _impl
from paddlescience_b200 import *  # noqa: F401,F403
from paddlescience_b200 import __all__ as _all

for _name in ("arch", "autodiff", "constraint", "data", "equation", "geometry", "loss", "metric", "optimizer", "solver", "utils",
              "validate"):
    _sys.modules[f"ppsci.{_name}"] = getattr(_impl, _name)
_sys.modules["ppsci.loss.mtl"] = _impl.loss.mtl
_sys.modules["ppsci.utils.logger"] = _impl.utils.logger
_sys.modules["ppsci.utils.misc"] = _impl.utils.misc
_sys.modules["ppsci.utils.symbolic"] = _impl.utils.symbolic
_sys.modules["ppsci.optimizer.lr_scheduler"] = _impl.optimizer.lr_scheduler
_sys.modules["ppsci.data.dataset"] = _impl.data.dataset
__all__ = list(_all)
