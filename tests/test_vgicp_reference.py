"""FastVGICP parity against the REFERENCE ITSELF: fast_gicp's unmodified fast_vgicp.cpp and pybind11 module, whose outputs
on every case of tests/vgicp_cases.py are kept as golden records in tests/golden/vgicp_ref_cases.npz
(tests/golden/make_vgicp_golden.py; tests/refgold.py).

  * CPU (`-m "not gpu"`): the numpy restatement of create_voxelmap (tests/vgicp_model.py), fed the CPU oracle's per-point
    covariances, reproduces the reference's voxel statistics.
  * GPU (`-m gpu`): pygicp.FastVGICP (CUDA, through the C ABI) against the reference on every case.
Bars: voxel means bit-exact (compared as sets sorted by mean); voxel covariances within 1e-13 of their largest entry (the
per-point covariances of the reference's Eigen code and of ours differ in the last bits); pose within 1e-6; final
Hessian within 1e-9 relative."""
import os

import numpy as np
import pytest

from gs_icp_slam_b200 import synthetic as S
from tests import vgicp_cases as cases
from tests import vgicp_model as VM
from tests.refgold import Record

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden", "vgicp_ref_cases.npz")


def _check_voxels(rec, out, suffix=""):
    rec.exact("vmean" + suffix, out["vmean" + suffix])
    err = rec.rel_err("vcov" + suffix, out["vcov" + suffix])
    assert err <= 1e-13, ("vcov" + suffix, err)


# ------------------------------------------------------------------------------------------------- CPU: model pin
def _oracle_target(setup):
    from oracle import gicp_oracle as G

    o = G.FastGICP()
    o.set_max_knn_distance(99999)
    setup(o)
    return o.get_target_covariances()


def _kitti_target():
    k = np.load(os.path.join(HERE, "golden", "gicp_kitti_pair.npz"))

    def setup(o):
        o.set_input_target(k["target"])
        o.calculate_target_covariance()

    return k["target"], _oracle_target(setup)


def _c3_target():
    g = S.gaussian_map(100000, 3)

    def setup(o):
        o.set_input_target(g["means3D"].astype(np.float64))
        o.set_target_covariances_fromqs(g["rotations"].reshape(-1), g["scales"].reshape(-1))

    return g["means3D"], _oracle_target(setup)


def _c1_target():
    tgt, _, _ = S.gicp_pair(4000, 4000)

    def setup(o):
        o.set_input_target(tgt)
        o.set_target_filter(len(tgt), np.arange(1, len(tgt) + 1, dtype=np.int32))
        o.calculate_target_covariance_with_filter()

    return tgt, _oracle_target(setup)


def _lattice_target():
    tgt = cases.lattice_target()

    def setup(o):
        o.set_input_target(tgt)
        o.calculate_target_covariance()

    return tgt, _oracle_target(setup)


@pytest.mark.parametrize("case,target,res", [
    ("kitti_r1.0_d1", _kitti_target, 1.0), ("kitti_r0.5_d1", _kitti_target, 0.5), ("c3_r0.05", _c3_target, 0.05),
    ("c3_r0.1", _c3_target, 0.1), ("c1_swap", _c1_target, 0.25), ("lattice", _lattice_target, 0.25)])
def test_model_voxel_statistics_match_reference(case, target, res):
    xyz, covs = target()
    m = VM.create_voxelmap(np.asarray(xyz, np.float32), covs, res)
    mean, cov = VM.sort_by_mean(*VM.as_reference_lists(m))
    _check_voxels(Record(GOLD, case), dict(vmean=mean, vcov=cov.reshape(-1, 16)))


# ------------------------------------------------------------------------------------------------- GPU: CUDA vs reference
@pytest.mark.gpu
@pytest.mark.parametrize("case", list(cases.CASES))
def test_fastvgicp_matches_reference(cuda, case):
    import pygicp

    fn, kw, posed = cases.CASES[case]
    out = fn(pygicp.FastVGICP, **kw)
    rec = Record(GOLD, case)
    for k, v in out.items():
        if k.startswith("vmean"):
            _check_voxels(rec, out, k[len("vmean"):])
        elif k.startswith("vcov"):
            continue  # with its vmean
        elif not posed:
            continue
        elif k.startswith("pose"):
            ref = rec.full(k)
            assert v.dtype == ref.dtype and np.abs(v.astype(np.float64) - ref).max() <= 1e-6, (k, np.abs(v - ref).max())
        elif k.startswith("H"):
            ref = rec.full(k)
            assert np.abs(v - ref).max() <= 1e-9 * np.abs(ref).max(), (k, np.abs(v - ref).max() / np.abs(ref).max())
        else:
            raise AssertionError(f"unclassified key {k}")
    if case == "no_overlap":  # the reference returns the guess and a zero Hessian
        assert not out["H"].any() and np.array_equal(out["pose"][:3, 3], np.float32([0.01, -0.02, 0.03]))
