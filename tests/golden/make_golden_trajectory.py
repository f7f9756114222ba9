"""Generates trajectory_viewer.json, the fixture of tests/test_gpu_trajectory.py: a 40-frame camera path (two
keyframes, 40 frames apart, with the "dynamic" timestep starting at 5 of 8 so that it clamps at 7) and the
trajectory.json the REAL reference local viewer (/root/reference local_viewer.py, read-only) exports for it, run on the
CPU with its GUI stubbed as tests/test_host_trajectory.py stubs it.  The keyframes are stored with their dtypes
(rot float64, look_at / radius / fovy float32), so the GPU test rebuilds the same path.

    python tests/golden/make_golden_trajectory.py
"""
import json
import os
import sys
import tempfile
from pathlib import Path
from types import SimpleNamespace

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.abspath(os.path.join(HERE, "..", ".."))
sys.path.insert(0, ROOT)
from gaussianavatars_b200 import trajectory as TR  # noqa: E402
from tests import test_host_trajectory as HT  # noqa: E402

W, H, T, START = 400, 304, 8, 5


def keyframes():
    from scipy.spatial.transform import Rotation
    rot = Rotation.from_euler("y", [[-25.0], [30.0]], degrees=True).as_matrix()
    return [TR.keyframe(rot[0], np.array([0.0, 0.01, 0.0], dtype=np.float32), 1.0, 20.0, 40),
            TR.keyframe(rot[1], np.array([0.005, -0.01, 0.0], dtype=np.float32), 0.9, 22.0, 40)]


def main():
    lv, _ = HT._reference()
    kfs = keyframes()
    with tempfile.TemporaryDirectory() as tmp:
        tmp = Path(tmp)
        ref = HT._ref_json(T, tmp / "transforms_test.json")
        v = HT._viewer(kfs, W, H, 0, "opencv", tmp, T=T, timestep=START, dynamic=True, ref_json=ref)
        lv.time = SimpleNamespace(sleep=lambda s: setattr(v, "need_update", False), strftime=lambda fmt: "export")
        lv.Image = SimpleNamespace(fromarray=lambda a: SimpleNamespace(save=lambda p: None))
        v.export_trajectory()
        traj = json.loads((tmp / "viewer" / "export" / "trajectory.json").read_text())
        ref_dict = json.loads(ref.read_text())
    out = {"width": W, "height": H, "num_timesteps": T, "start_timestep": START, "ref_json": ref_dict,
           "keyframes": [{k: (np.asarray(v).tolist() if k != "interval" else v) for k, v in kf.items()} for kf in kfs],
           "trajectory": traj}
    with open(os.path.join(HERE, "trajectory_viewer.json"), "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
