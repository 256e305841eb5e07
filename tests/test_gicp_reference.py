"""GICP parity against the REFERENCE ITSELF: fast_gicp's unmodified sources + its own pybind11 module (built by
`make -C oracle ref` against the vendored Eigen and oracle/pcl_shim), whose outputs on every case are kept as golden
records in tests/golden/fastgicp_cases.npz (tests/golden/make_reference_cpu_golden.py; tests/refgold.py).

  * CPU (`-m "not gpu"`): the oracle restatement (oracle/gicp_oracle.cpp) is pinned to the real fast_gicp on C1, on
    the C3 tracker shape (12 416-point frames vs a Gaussian-map target from (q, s), estimated-pose seeding), on the
    reference's KITTI fixture, on the bindings the SLAM never calls and on duplicates / outliers, and to golden vectors
    of the real fast_gicp (tests/golden/gicp_fastgicp_ref.npz).
  * GPU (`-m gpu`): the CUDA tracker (pygicp drop-in, through the C ABI) against the real fast_gicp on the same cases.
Bars: neighbour indices, squared distances and the float32 rotation/scale exports bit-exact; pose within 1e-6;
final 6x6 normal equations within 1e-9 relative."""
import os

import numpy as np
import pytest

from tests import gicp_cases as cases
from tests.refgold import Record

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden", "gicp_fastgicp_ref.npz")
CASES = os.path.join(HERE, "golden", "fastgicp_cases.npz")


def _oracle():
    from oracle import gicp_oracle as G

    return G.FastGICP()


def _cuda():
    import pygicp

    return pygicp.FastGICP()


def _ref(case):
    return Record(CASES, case)


# ------------------------------------------------------------------------------------------------- CPU: oracle pin
def test_oracle_matches_fast_gicp_c1():
    cases.compare_golden(cases.c1(_oracle), _ref("c1"))


def test_oracle_matches_fast_gicp_tracker_c3_shape():
    # 100k-Gaussian target keeps the CPU suite short; the GPU test runs the full 300k
    a = cases.tracker_c3(_oracle, P=100000)
    cases.compare_golden(a, _ref("tracker_c3_100k"))
    assert np.abs(a["pose3"] - a["gt_last"]).max() < 2e-2


def test_oracle_matches_fast_gicp_kitti():
    a, b = cases.kitti(_oracle), _ref("kitti")
    cases.compare_golden(a, b)
    pose, rel = b.full("pose").astype(np.float64), a["relative"]
    assert np.linalg.norm(pose[:3, 3] - rel[:3, 3]) < 0.05  # the reference's own acceptance bound (gicp_test.cpp:55-56)
    dR = pose[:3, :3] @ rel[:3, :3].T
    assert np.degrees(np.arccos(min(1.0, (np.trace(dR) - 1) / 2))) < 1.0


def test_oracle_matches_fast_gicp_golden():
    """Golden vectors produced by the real fast_gicp build (tests/golden/make_gicp_ref_golden.py): the pin that travels."""
    g = np.load(GOLD)
    a = cases.c1(_oracle, n=4000)
    ref = {k[len("c1_"):]: g[k] for k in g.files if k.startswith("c1_")}
    cases.compare({k: a[k] for k in ref}, ref)
    a = cases.tracker_c3(_oracle, P=20000, frames=(1, 2), keyframe_at=1)
    ref = {k[len("trk_"):]: g[k] for k in g.files if k.startswith("trk_")}
    cases.compare({k: a[k] for k in ref}, ref)


@pytest.mark.parametrize("kw", [dict(), dict(k=10), dict(max_knn=0.05)], ids=["k20", "k10", "knn-radius-0.05"])
def test_oracle_matches_fast_gicp_on_the_bindings_the_slam_never_calls(request, kw):
    """withz covariances + z values, set_correspondence_randomness, a finite k-NN radius, get_fitness_score and
    swap_source_and_target (main.cpp:169,172,203,205,228,246-253): the oracle the CUDA path is tested against
    (tests/test_gicp_gpu.py::test_unused_by_slam_bindings_match_oracle) is itself pinned to the real fast_gicp here."""
    a, b = _ref("unused_bindings_" + request.node.callspec.id), cases.unused_bindings(_oracle, **kw)
    for k in ("tgt_rots", "tgt_scales_z", "src_rots", "src_scales", "corr", "sqd", "corr_swapped", "sqd_swapped"):
        a.exact(k, b[k])
    assert np.array_equal(a.full("pose"), b["pose"]) and np.array_equal(a.full("pose_swapped"), b["pose_swapped"])
    assert np.abs(a.full("H") - b["H"]).max() <= 1e-12 * np.abs(a.full("H")).max()
    # getFitnessScore lives in PCL's Registration base class (here: oracle/pcl_shim): float transform of the cloud, 1-NN
    assert np.allclose(a.full("fitness"), b["fitness"], rtol=2e-6, atol=0)


def test_oracle_matches_fast_gicp_with_duplicates_and_outliers():
    """Ties (duplicated points in both clouds) and source points with no correspondence within max_corr (-1 rows)."""
    a, b = _ref("duplicates_and_outliers"), cases.duplicates_and_outliers(_oracle)
    cases.compare_golden(b, a)
    assert (b["corr"][:50] == -1).all() and np.array_equal(a.full("pose"), b["pose"])


# ------------------------------------------------------------------------------------------------- GPU: product pin
@pytest.mark.gpu
def test_cuda_matches_fast_gicp_c1(cuda):
    a = cases.c1(_cuda)
    cases.compare_golden(a, _ref("c1"))
    assert np.abs(a["pose"] - a["T_gt"]).max() < 1e-3


@pytest.mark.gpu
def test_cuda_matches_fast_gicp_tracker_c3(cuda):
    """Full C3 tracker shape: 12 416-point frames against the 300k-Gaussian target."""
    a = cases.tracker_c3(_cuda)
    cases.compare_golden(a, _ref("tracker_c3"))
    assert np.abs(a["pose3"] - a["gt_last"]).max() < 2e-2


@pytest.mark.gpu
def test_cuda_matches_fast_gicp_kitti(cuda):
    cases.compare_golden(cases.kitti(_cuda), _ref("kitti"))


@pytest.mark.gpu
def test_cuda_matches_fast_gicp_golden(cuda):
    g = np.load(GOLD)
    a = cases.c1(_cuda, n=4000)
    ref = {k[len("c1_"):]: g[k] for k in g.files if k.startswith("c1_")}
    cases.compare({k: a[k] for k in ref}, ref)
