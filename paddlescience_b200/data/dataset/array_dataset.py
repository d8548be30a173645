"""Array datasets that define the batch layout of the hot path: a dict of ``[N, 1]`` columns
(reference: ppsci/data/dataset/array_dataset.py:29-231)."""
from __future__ import annotations

from typing import Callable, Dict, Optional

import numpy as np
import torch


def _to_tensor_dict(d: Optional[Dict[str, np.ndarray]], dtype=None):
    if d is None:
        return None
    return {k: torch.as_tensor(np.asarray(v)) if dtype is None else torch.as_tensor(np.asarray(v)).to(dtype)
            for k, v in d.items()}


class NamedArrayDataset:
    """Map-style dataset indexed per sample or per batch of indices (array_dataset.py:29-85)."""

    batch_index: bool = True

    def __init__(self, input: Dict[str, np.ndarray], label: Optional[Dict[str, np.ndarray]] = None,
                 weight: Optional[Dict[str, np.ndarray]] = None, transforms=None):
        self.input = input
        self.label = {} if label is None else label
        self.weight = {} if weight is None else weight
        self.input_keys = tuple(input.keys())
        self.label_keys = tuple(self.label.keys())
        self.transforms = transforms
        self._len = len(next(iter(input.values())))

    def __getitem__(self, idx):
        item = ({k: v[idx] for k, v in self.input.items()}, {k: v[idx] for k, v in self.label.items()},
                {k: v[idx] for k, v in self.weight.items()})
        if self.transforms is not None:
            item = self.transforms(*item)
        return item

    def __len__(self):
        return self._len


class IterableNamedArrayDataset:
    """Full-batch dataset: every iteration yields the whole (device-resident) set
    (array_dataset.py:88-151)."""

    batch_index: bool = False

    def __init__(self, input: Dict[str, np.ndarray], label: Optional[Dict[str, np.ndarray]] = None,
                 weight: Optional[Dict[str, np.ndarray]] = None, transforms=None):
        self.input = _to_tensor_dict(input)
        self.label = _to_tensor_dict(label) if label is not None else {}
        self.weight = _to_tensor_dict(weight, torch.get_default_dtype()) if weight is not None else None
        self.input_keys = tuple(input.keys())
        self.label_keys = tuple(self.label.keys())
        self._len = len(next(iter(self.input.values())))
        self.transforms = transforms

    @property
    def num_samples(self):
        return self._len

    def to(self, device):
        self.input = {k: v.to(device) for k, v in self.input.items()}
        self.label = {k: v.to(device) for k, v in self.label.items()}
        if self.weight is not None:
            self.weight = {k: v.to(device) for k, v in self.weight.items()}
        return self

    def __iter__(self):
        if callable(self.transforms):
            yield self.transforms(self.input, self.label, self.weight)
        else:
            yield self.input, self.label, self.weight

    def __len__(self):
        return 1


class ContinuousNamedArrayDataset:
    """Endless sampler dataset: user callables produce a fresh numpy batch each step
    (array_dataset.py:154-231)."""

    batch_index: bool = False

    def __init__(self, input: Callable, label: Callable, weight: Optional[Callable] = None, transforms=None):
        self.input_fn = input
        self.input_keys = tuple(self.input_fn().keys())
        self.label_fn = label
        self.label_keys = tuple(self.label_fn(self.input_fn()).keys())
        self.weight_fn = weight
        self.transforms = transforms

    @property
    def num_samples(self):
        raise NotImplementedError("ContinuousNamedArrayDataset has no fixed number of samples.")

    def __iter__(self):
        while True:
            inp = self.input_fn()
            lab = self.label_fn(inp)
            wt = self.weight_fn(inp, lab) if callable(self.weight_fn) else None
            if callable(self.transforms):
                inp, lab, wt = self.transforms(inp, lab, wt)
            yield _to_tensor_dict(inp), _to_tensor_dict(lab), _to_tensor_dict(wt)

    def __len__(self):
        return 1


class DeviceUniformSampler:
    """``input`` callable for ``ContinuousNamedArrayDataset`` that draws its batch ON the device: ``n`` points uniform in
    the box ``[lo, hi]`` per call (SURVEY section 8(f) rank 4; the reference draws with numpy on the host and copies every
    step, array_dataset.py:208-228).  Counter-based Philox stream (``ppsci_b200_sample_uniform``): call ``k`` uses the
    counter range ``[k n, (k + 1) n)``, so a run is reproducible from ``seed`` alone; under data parallelism give every
    rank the same seed and ``rank_offset = rank`` (disjoint counter ranges)."""

    def __init__(self, keys, lo, hi, n: int, seed: int = 42, dtype=None, device="cuda", rank_offset: int = 0, world: int = 1):
        import torch

        self.keys = tuple(keys)
        self.lo = [float(v) for v in lo]
        self.hi = [float(v) for v in hi]
        if not (len(self.keys) == len(self.lo) == len(self.hi)):
            raise ValueError("keys, lo and hi must have the same length")
        self.n, self.seed = int(n), int(seed)
        self.dtype = dtype or torch.float32
        self.device = torch.device(device)
        self.rank_offset, self.world = int(rank_offset), int(world)
        self.calls = 0

    def __call__(self):
        import ctypes as C

        import torch

        from ...engine import binding as B

        lib = B.get_library()
        cols = [torch.empty(self.n, 1, dtype=self.dtype, device=self.device) for _ in self.keys]
        nd = len(self.keys)
        lo = (C.c_double * nd)(*self.lo)
        hi = (C.c_double * nd)(*self.hi)
        ptrs = (C.c_void_p * nd)(*[c.data_ptr() for c in cols])
        offset = (self.calls * self.world + self.rank_offset) * self.n
        stream = torch.cuda.current_stream(self.device).cuda_stream if self.device.type == "cuda" else 0
        rc = lib.lib.ppsci_b200_sample_uniform(B.F64 if self.dtype == torch.float64 else B.F32, self.seed, offset, self.n, nd, lo, hi,
                                               ptrs, stream)
        lib.check(rc, "sample_uniform")
        self.calls += 1
        return dict(zip(self.keys, cols))


class ChipHeatDataset:
    """The chip-heat operator dataset (array_dataset.py:234-312): sample ``idx`` is one cell of the cartesian product of
    the inputs named in ``index`` (point x source function x boundary type x boundary function), decoded as a
    mixed-radix number whose first digit varies fastest.  ``y`` follows ``x``'s digit; ``u_one`` (the source or
    boundary function at that point) is row ``len(input[data_type]) * i_x + i_{data_type}``; every other input key is
    indexed by its own digit.  Labels and weights are per-constraint constants, repeated for every sample.

    ``idx`` may be one index or an integer array: a batch is gathered in one vectorised pass (what the batch loader
    asks for), the same rows the reference's per-sample loop would collate."""

    batch_index: bool = True

    def __init__(self, input: Dict[str, np.ndarray], label: Dict[str, np.ndarray], index, data_type: str,
                 weight: Optional[Dict[str, np.ndarray]] = None, transforms=None):
        self.input = input
        self.label = label
        self.input_keys = tuple(input.keys())
        self.label_keys = tuple(label.keys())
        self.index = tuple(index)
        self.data_type = data_type
        self.weight = {} if weight is None else weight
        self.transforms = transforms

    def __getitem__(self, idx):
        quotient = np.asarray(idx, dtype=np.int64)
        digit = {}
        for k in dict.fromkeys(self.index):
            num = len(self.input[k])
            digit[k] = quotient % num
            quotient = quotient // num
        input_item = {}
        for key, v in self.input.items():
            if key == "y":
                input_item[key] = v[digit["x"]]
            elif key == "u_one":
                input_item[key] = v[len(self.input[self.data_type]) * digit["x"] + digit[self.data_type]]
            else:
                input_item[key] = v[digit[key]]
        if np.ndim(idx) == 0:
            label_item, weight_item = dict(self.label), dict(self.weight)
        else:
            n = len(idx)
            label_item = {k: np.repeat(np.asarray(v)[None], n, axis=0) for k, v in self.label.items()}
            weight_item = {k: np.repeat(np.asarray(v)[None], n, axis=0) for k, v in self.weight.items()}
        if self.transforms is not None:
            input_item, label_item, weight_item = self.transforms((input_item, label_item, weight_item))
        return input_item, label_item, weight_item

    def __len__(self):
        n = 1
        for k in self.index:
            n *= len(self.input[k])
        return n
