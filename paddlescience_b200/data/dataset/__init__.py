from .array_dataset import (ChipHeatDataset, ContinuousNamedArrayDataset, DeviceUniformSampler,
                            IterableNamedArrayDataset, NamedArrayDataset)

__all__ = ["NamedArrayDataset", "IterableNamedArrayDataset", "ContinuousNamedArrayDataset", "DeviceUniformSampler", "ChipHeatDataset",
           "build_dataset"]


def build_dataset(cfg):
    """ppsci/data/dataset/__init__.py — build a dataset from a dict with a ``name`` entry."""
    cfg = dict(cfg)
    name = cfg.pop("name")
    if name not in globals():
        raise NotImplementedError(f"dataset {name} is outside the hot path this framework covers")
    return globals()[name](**cfg)
