"""Golden data of tests/test_accel.py: the state dicts (keys in order, tensors), autoregressive orders and
masks of the flows `_flows` builds, as the UNMODIFIED reference builds them under torch.manual_seed(0).
The tests build the same flows with the engine's constructors, accelerate them and compare with these.
Run with the reference's source tree as the first argument:

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_accel.py <reference source tree>
"""

from __future__ import annotations

import sys
from pathlib import Path

import numpy as np

sys.dont_write_bytecode = True
HERE = Path(__file__).resolve().parent
sys.path.insert(0, sys.argv[1])
sys.path.insert(0, str(HERE.parent))
sys.path.insert(0, str(HERE.parent.parent))

import zuko  # noqa: E402
from test_accel import _flows  # noqa: E402


def main() -> None:
    out = {}
    for name, flow in _flows(zuko).items():
        sd = flow.state_dict()
        out[f"{name}/keys"] = np.array(list(sd), dtype=np.str_)
        for i, t in enumerate(sd.values()):
            out[f"{name}/sd/{i:03d}"] = t.detach().cpu().numpy()
        for i, t in enumerate(flow.transform.transforms):
            if getattr(t, "order", None) is not None:
                out[f"{name}/order/{i}"] = t.order.cpu().numpy()
                out[f"{name}/passes/{i}"] = np.array(t.passes)
                for j, m in enumerate(t.hyper):
                    if hasattr(m, "mask"):
                        out[f"{name}/mask/{i}/{j}"] = m.mask.cpu().numpy()
            elif hasattr(t, "passes"):
                out[f"{name}/passes/{i}"] = np.array(t.passes)
    np.savez_compressed(HERE / "accel_reference.npz", **out)


if __name__ == "__main__":
    main()
