"""The hand trajectory of MyoSuite's tutorial 6 (tutorials/data/6_trajectory.csv: time, then the 23 joint angles of myohand_pose in model
order at the model's 2 ms timestep) downsampled to every 5th frame, as float32.  Output: tests/golden/hand_trajectory.npz (qpos [T, 23],
dt), read by the computed-muscle-control test of tests/test_static_opt.py, which interpolates it back to the timestep with a cubic spline.
Run with a MyoSuite checkout (MYOSUITE_CHECKOUT=<its root>):  python tests/golden/make_hand_trajectory.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from myosuite_b200 import assets  # noqa: E402

EVERY = 5
src = os.path.join(os.environ.get("MYOSUITE_CHECKOUT", "."), "tutorials", "data", "6_trajectory.csv")
names = open(src).readline().strip().split(",")
data = np.loadtxt(src, delimiter=",", skiprows=1)
m = assets.load("myohand_pose")
assert names[0] == "time" and names[1:] == [m.id2name("joint", j) for j in range(m.njnt)] and m.nq == len(names) - 1
dt = float(np.median(np.diff(data[:, 0])))
assert abs(dt - m.opt_timestep) < 1e-12
q = data[::EVERY, 1:].astype(np.float32)
np.savez_compressed(os.path.join(HERE, "hand_trajectory.npz"), qpos=q, dt=np.float64(dt * EVERY))
print("hand_trajectory.npz: %d frames of %d joints every %.3f s (of %d at %.3f s)" % (q.shape[0], q.shape[1], dt * EVERY, len(data), dt))
