"""Generates the golden records of the reference's CPU code that the parity tests compare against (tests/refgold.py):
    fastgicp_cases.npz    fast_gicp's own tracker (oracle/_ref/fast_gicp) on every case of tests/gicp_cases.py that
                          tests/test_gicp_reference.py runs
    eigen_ref_calls.npz   the reference's vendored Eigen (oracle/_ref/libref_gicp_eigen.so): every call the tests of
                          tests/test_gicp_oracle.py make, with its outputs
    scene_ply_ref.npz     SHA-256 of the scene.ply bytes the reference's GaussianModel.save_ply writes
Needs the reference build of `make -C oracle ref` where the reference's sources are present (its `ref_ext` step also
installs the reference's SLAM scripts into oracle/_ref/gs_icp_slam, which scene_ply() imports); no GPU:
    python tests/golden/make_reference_cpu_golden.py"""
import ctypes as C
import hashlib
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")


def fastgicp_cases():
    from oracle import ref_gicp
    from tests import gicp_cases as cases
    from tests import refgold

    make = ref_gicp.FastGICP
    runs = {"c1": cases.c1(make), "tracker_c3_100k": cases.tracker_c3(make, P=100000), "tracker_c3": cases.tracker_c3(make),
            "kitti": cases.kitti(make), "duplicates_and_outliers": cases.duplicates_and_outliers(make)}
    for name, kw in (("k20", dict()), ("k10", dict(k=10)), ("knn-radius-0.05", dict(max_knn=0.05))):
        runs["unused_bindings_" + name] = cases.unused_bindings(make, **kw)
    out = {}
    for name, res in runs.items():
        out.update(refgold.pack(name, res, sample=False))  # poses and H are kept whole; everything else is compared bit-exact
    np.savez_compressed(os.path.join(GOLD, "fastgicp_cases.npz"), **out)


def eigen_calls():
    from tests import refgold
    from tests import test_gicp_oracle as T

    lib = C.CDLL(os.path.join(ROOT, "oracle", "_ref", "libref_gicp_eigen.so"))
    out = {}
    for name in ("test_svd_and_quaternion_match_eigen", "test_quaternion_of_reflection_matches_eigen",
                 "test_ldlt_and_so3_exp_match_eigen", "test_covariance_pipeline_matches_eigen", "test_cov_from_qs_quirk_matches_eigen",
                 "test_linearize_matches_eigen_per_point"):
        rec = refgold.EigenRecorder(lib)
        getattr(T, name)(rec)
        out.update(rec.arrays(name))
    np.savez_compressed(os.path.join(GOLD, "eigen_ref_calls.npz"), **out)


def scene_ply():
    from tests import test_scene_ply as T

    out = {}
    for degree in (0, 3):
        with tempfile.TemporaryDirectory() as d:
            path = T.reference_save_ply(os.path.join(ROOT, "oracle", "_ref", "gs_icp_slam"), d, degree)
            out[f"degree{degree}"] = np.frombuffer(hashlib.sha256(open(path, "rb").read()).digest(), np.uint8)
    np.savez_compressed(os.path.join(GOLD, "scene_ply_ref.npz"), **out)


if __name__ == "__main__":
    fastgicp_cases()
    eigen_calls()
    scene_ply()
    for f in ("fastgicp_cases.npz", "eigen_ref_calls.npz", "scene_ply_ref.npz"):
        print(f, os.path.getsize(os.path.join(GOLD, f)))
