"""Generates tests/golden/lr_schedule.npz by IMPORTING the real reference learning-rate schedule
(utils/general_utils.py get_expon_lr_func) with the default OptimizationParams values (arguments/__init__.py: the
`xyz` schedule of scene/gaussian_model.py:224-227 at spatial_lr_scale = 1) and evaluating it at a spread of
iterations.  A second schedule adds a delay (lr_delay_steps > 0), which the default leaves off, so that the fixture
also covers the reference's cosine warm-up.  The fixture travels to the GPU box; the reference does not.

    python tests/golden/make_golden_lr.py
"""
import os
import sys
from argparse import ArgumentParser

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.abspath(os.path.join(HERE, "..", ".."))
sys.path.insert(0, ROOT)

from tests import ref_import  # noqa: E402

ITERATIONS = np.array([1, 2, 3, 10, 100, 999, 1000, 1001, 5000, 29_999, 30_000, 123_457, 299_999, 300_000, 599_999,
                       600_000, 600_001, 750_000], dtype=np.int64)


def main():
    ref_import.prepare()
    from arguments import OptimizationParams  # noqa: E402  (REAL reference code)
    from utils.general_utils import get_expon_lr_func  # noqa: E402

    op = OptimizationParams(ArgumentParser())
    schedules = {
        "default": dict(lr_init=op.position_lr_init, lr_final=op.position_lr_final, lr_delay_steps=0,
                        lr_delay_mult=op.position_lr_delay_mult, max_steps=op.position_lr_max_steps),
        "delayed": dict(lr_init=op.position_lr_init, lr_final=op.position_lr_final, lr_delay_steps=5000,
                        lr_delay_mult=op.position_lr_delay_mult, max_steps=op.position_lr_max_steps),
    }
    out = {"iterations": ITERATIONS}
    for name, kw in schedules.items():
        f = get_expon_lr_func(**kw)
        out[f"{name}_lr"] = np.array([float(f(int(it))) for it in ITERATIONS], dtype=np.float64)
        out[f"{name}_args"] = np.array([kw["lr_init"], kw["lr_final"], kw["lr_delay_steps"], kw["lr_delay_mult"],
                                        kw["max_steps"]], dtype=np.float64)
    np.savez(os.path.join(HERE, "lr_schedule.npz"), **out)
    for k, v in out.items():
        print(k, v)


if __name__ == "__main__":
    main()
