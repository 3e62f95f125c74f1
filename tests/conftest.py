import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; select with -m gpu)")


@pytest.fixture(scope="session", autouse=True)
def _build_everything():
    """Build the oracle (CPU checker) and the native library once per session."""
    import oracle

    oracle.build()
    import build_native as b

    b.build_native()
    b.build_host_cpp()


@pytest.fixture(scope="session")
def pair02():
    d = np.load(os.path.join(GOLDEN, "pair_0p2.npz"))
    return d["target"], d["source"]


@pytest.fixture(scope="session")
def pair01():
    d = np.load(os.path.join(GOLDEN, "pair_0p1.npz"))
    return d["target"], d["source"]


@pytest.fixture(scope="session")
def relative_pose():
    return np.loadtxt(os.path.join(GOLDEN, "relative.txt"))


def pose_error(T_ref, T):
    """(translation error [m], rotation error [rad]) of T against T_ref -- gicp_test.cpp:75-80."""
    d = np.linalg.inv(np.asarray(T_ref, dtype=np.float64)) @ np.asarray(T, dtype=np.float64)
    t = float(np.linalg.norm(d[:3, 3]))
    # angle from sin and cos (atan2): arccos of the trace alone turns a 1e-7 non-orthonormality of a float32 pose matrix
    # (pcl::Registration keeps Matrix4f) into sqrt(2e-7) = 4e-4 rad
    R = d[:3, :3]
    s = 0.5 * np.linalg.norm([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
    c = (np.trace(R) - 1.0) / 2.0
    return t, float(np.arctan2(s, c))


def random_pose(rng, max_angle, max_trans):
    w = rng.normal(size=3)
    w = w / np.linalg.norm(w) * rng.uniform(0, max_angle)
    th = np.linalg.norm(w)
    K = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
    R = np.eye(3) + (np.sin(th) / th) * K + ((1 - np.cos(th)) / th**2) * K @ K if th > 0 else np.eye(3)
    T = np.eye(4)
    T[:3, :3] = R
    T[:3, 3] = rng.uniform(-max_trans, max_trans, size=3)
    return T
