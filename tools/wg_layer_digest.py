"""SHA-256 digests of everything the wgmma forward / dx kernel (k_wg_layer) writes in one fused call.

For three seeded calls (the flagship shape 6 x 256 with the Navier-Stokes layout at a ragged point count that takes
many persistent passes, a 128-wide Lay4444 call and a 160-wide call, i.e. an odd number of 32-column blocks) the
pre-activation jets Z_l of every hidden layer, the output jets Y, the output adjoints Ybar and the two hidden adjoints
that survive the call (Zbar_1, Zbar_2) are read back from the plan's workspace and hashed.  A change to the kernel that
keeps the order in which every accumulator element receives its products leaves every digest as it was.

    python tools/wg_layer_digest.py [--lib PATH ...]

With several --lib the libraries' digests are printed side by side and every row says whether they agree.  Ybar comes
from the head kernel, not from k_wg_layer; it is listed because the Zbar digests can only agree where it does.  The
weight gradient goes through atomicAdd and is not expected to be bitwise stable, so it is not hashed.  Needs an H100.
"""
from __future__ import annotations

import argparse
import hashlib
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from paddlescience_b200.engine import binding  # noqa: E402
from tests.layer_ref import run_fused  # noqa: E402

CASES = [
    ("cfg3 Lay22 6x256 n=49999", "Lay22", [256] * 6, 49_999),
    ("Lay4444 3x128 n=5001", "Lay4444", [128] * 3, 5_001),
    ("Lay22 3x160 n=10001", "Lay22", [160] * 3, 10_001),
]


def digests(library) -> dict:
    out = {}
    for name, layout, hidden, n in CASES:
        plan, _, _, views = run_fused(layout, hidden, n, library=library)
        if not plan.uses_tcgen05:
            raise RuntimeError(f"{name}: the plan does not run on the tensor-core kernels")
        torch.cuda.synchronize()
        for key, v in views.items():
            out[f"{name}  {key}"] = hashlib.sha256(v.contiguous().cpu().numpy().tobytes()).hexdigest()[:16]
    return out


def main() -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--lib", action="append", default=None, help="native library to run (repeatable); default: the tree's")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("wg_layer_digest needs an H100: the engine has no CPU fallback")
    paths = args.lib or [binding.default_library_path()]
    cols = [digests(binding.Library(p)) for p in paths]
    for i, p in enumerate(paths):
        print(f"lib{i} = {p}")
    same = True
    for key in cols[0]:
        row = [c[key] for c in cols]
        ok = all(d == row[0] for d in row)
        same &= ok
        print(f"{key:<34} " + "  ".join(row) + ("" if len(cols) == 1 else "  same" if ok else "  DIFFERENT"))
    return 0 if same else 1


if __name__ == "__main__":
    sys.exit(main())
