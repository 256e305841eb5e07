"""pygicp.FastVGICP on the GPU against the float64 numpy restatement of fast_gicp's FastVGICP (tests/vgicp_model.py), fed
the GPU's own per-point covariances: the voxel map (means bit-exact), linearize and compute_error at several poses (H, b
and the error within 1e-9 relative), determinism, map rebuilds, CUDA-tensor inputs, the error paths, and a FastGICP run
that a live FastVGICP leaves untouched."""
import numpy as np
import pytest

from gs_icp_slam_b200 import synthetic as S
from tests import vgicp_model as VM

pytestmark = pytest.mark.gpu


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


def _small_rot(deg, axis, t):
    T = np.eye(4)
    T[:3, :3] = S.rotation_about(axis, np.radians(deg))
    T[:3, 3] = t
    return T


def _vgicp(tgt, src, res=0.25, method="DIRECT1"):
    import pygicp

    r = pygicp.FastVGICP()
    r.set_max_knn_distance(99999)
    r.set_resolution(res)
    r.set_neighbor_search_method(method)
    r.set_input_target(tgt)
    r.calculate_target_covariance()
    r.set_input_source(src)
    r.calculate_source_covariance()
    return r


def _check_map(r, tgt, res):
    m = VM.create_voxelmap(np.asarray(tgt, np.float32), r.get_target_covariances(), res)
    mu, C = r.get_voxel_mean_cov()
    assert len(mu) == len(m["keys"]) and all(x.shape == (4,) and x.dtype == np.float64 for x in mu)
    assert all(c.shape == (4, 4) and c.dtype == np.float64 for c in C)
    em, ec = VM.as_reference_lists(m)
    assert np.array_equal(np.array(mu), em)  # same key order, bit-exact means
    assert np.abs(np.array(C) - ec).max() <= 1e-13 * np.abs(ec).max()
    return m


@pytest.mark.parametrize("method,n_off", [("DIRECT1", 1), ("DIRECT7", 7), ("DIRECT27", 27)])
def test_linearize_and_error_match_model(cuda, method, n_off):
    tgt, src, _ = S.gicp_pair(6000, 5000)
    r = _vgicp(tgt, src, 0.25, method)
    src32 = np.asarray(src, np.float32)
    covs = r.get_source_covariances()
    poses = [np.eye(4), _small_rot(1.0, (0, 0, 1), (0.02, -0.01, 0.0)), _small_rot(3.0, (1, 1, 0), (-0.05, 0.03, 0.02))]
    for P in poses:
        H, b, e = r.linearize(P)
        m = _check_map(r, tgt, 0.25)
        Hm, bm, em = VM.linearize(m, src32, covs, P, n_off)
        assert np.array_equal(H, H.T)
        assert _rel(H, Hm) <= 1e-9 and _rel(b, bm) <= 1e-9 and abs(e - em) <= 1e-9 * abs(em), (method, _rel(H, Hm), _rel(b, bm))
        # compute_error keeps the pairs and M of the linearisation pose P, only the error vector moves
        for Q in poses:
            eq = r.compute_error(Q)
            assert abs(eq - VM.compute_error(m, src32, covs, P, Q, n_off)) <= 1e-9 * max(abs(em), 1e-300)
        assert r.compute_error(P) == e  # same pairs, same M, same arithmetic


def test_align_is_deterministic_and_converges(cuda):
    tgt, src, T = S.gicp_pair(8000, 6000)
    out = []
    for _ in range(2):
        r = _vgicp(tgt, src, 0.25, "DIRECT7")
        out.append((r.align(np.eye(4, dtype=np.float32)), r.get_final_hessian()))
    assert np.array_equal(out[0][0], out[1][0]) and np.array_equal(out[0][1], out[1][1])
    assert np.abs(out[0][0] - T).max() < 5e-3
    with pytest.raises(Exception):
        r.get_source_correspondence()  # no point-to-point correspondences, as a FastGICP with stale ones


def test_map_is_rebuilt(cuda):
    tgt, src, _ = S.gicp_pair(6000, 4000)
    tgt2, _, _ = S.gicp_pair(5000, 10, seed_t=7, scale=1.3)
    r = _vgicp(tgt, src, 0.25)
    assert r.get_voxel_mean_cov() == ([], [])  # no map before the first align
    r.align()
    _check_map(r, tgt, 0.25)
    # set_input_target drops the map; the next align builds it from the new target
    r.set_input_target(tgt2)
    assert r.get_voxel_mean_cov() == ([], [])
    r.calculate_target_covariance()
    r.align()
    _check_map(r, tgt2, 0.25)
    # new target covariances from (q, s)
    g = S.gaussian_map(3000, 5)
    r.set_input_target(g["means3D"].astype(np.float64))
    r.set_target_covariances_fromqs(g["rotations"].reshape(-1), g["scales"].reshape(-1))
    r.align()
    _check_map(r, g["means3D"], 0.25)
    # calculate_target_covariance_with_filter compacts the target to its trackable points
    r.set_input_target(tgt)
    keep = np.zeros(len(tgt), np.int32)
    keep[::2] = np.arange(1, (len(tgt) + 1) // 2 + 1, dtype=np.int32)
    r.set_target_filter(int(keep.max()), keep)
    r.calculate_target_covariance_with_filter()
    r.align()
    _check_map(r, tgt[::2], 0.25)
    # a new resolution takes effect at the next align
    r.set_resolution(0.5)
    _check_map(r, tgt[::2], 0.25)
    r.align()
    _check_map(r, tgt[::2], 0.5)
    # after a swap the former source is the target
    r.swap_source_and_target()
    assert r.get_voxel_mean_cov() == ([], [])
    r.set_source_filter(len(tgt[::2]), np.arange(1, len(tgt[::2]) + 1, dtype=np.int32))
    r.align()
    _check_map(r, src, 0.5)


def test_cuda_tensor_inputs_match_numpy(cuda):
    import torch

    g = S.gaussian_map(20000, 3)
    pts, tr = S.tracker_cloud(S.raycast_depth(S.trajectory_pose(1, 200), S.TUM)[0], S.TUM)
    guess = S.trajectory_pose(0, 200).astype(np.float32)
    outs = []
    for dev in (False, True):
        import pygicp

        r = pygicp.FastVGICP()
        r.set_max_knn_distance(99999)
        r.set_resolution(0.05)
        f = S.trackable_filter(len(pts), tr)
        if dev:
            r.set_input_target(torch.from_numpy(g["means3D"]).to(cuda))
            r.set_target_covariances_fromqs(torch.from_numpy(g["rotations"]).to(cuda), torch.from_numpy(g["scales"]).to(cuda))
            r.set_input_source(torch.from_numpy(np.asarray(pts, np.float32)).to(cuda))
            r.set_source_filter(len(tr), torch.from_numpy(np.asarray(f)).to(cuda))
        else:
            r.set_input_target(g["means3D"])
            r.set_target_covariances_fromqs(g["rotations"].reshape(-1), g["scales"].reshape(-1))
            r.set_input_source(np.asarray(pts, np.float32))
            r.set_source_filter(len(tr), f)
        outs.append((r.align(guess), r.get_final_hessian(), np.array(r.get_voxel_mean_cov()[0])))
    for a, b in zip(*outs):
        assert np.array_equal(a, b)


def test_error_paths(cuda, capfd):
    import pygicp
    from gs_icp_slam_b200._lib import GsicpError

    r = pygicp.FastVGICP()
    for bad in (0.0, -1.0, float("nan"), float("inf")):
        with pytest.raises(GsicpError):
            r.set_resolution(bad)
    with pytest.raises(ValueError):
        r.set_neighbor_search_method("DIRECT_RADIUS")
    r.set_neighbor_search_method("DIRECT7")
    capfd.readouterr()
    r.set_neighbor_search_method("NOPE")  # falls back to DIRECT1 with the reference's message
    assert "error: unknown neighbor search method NOPE" in capfd.readouterr().err
    with pytest.raises(GsicpError, match="one GPU"):
        r.set_shard(2, 0)
    with pytest.raises(GsicpError, match="one GPU"):
        r.set_comm(None)
    assert r.get_voxel_mean_cov() == ([], [])
    with pytest.raises(GsicpError):
        r.compute_error(np.eye(4))  # no linearize yet
    # a target whose voxel extent needs more than 21 bits on an axis
    tgt = np.array([[0.0, 0.0, 0.0], [3000.0, 0.0, 0.0], [0.0, 1.0, 0.0], [0.0, 0.0, 1.0]] * 5)
    tgt += np.random.default_rng(0).normal(0, 1e-3, tgt.shape)
    r.set_resolution(1e-3)
    r.set_input_target(tgt)
    r.calculate_target_covariance()
    r.set_input_source(tgt[:8])
    r.set_source_filter(8, np.arange(1, 9, dtype=np.int32))
    with pytest.raises(GsicpError, match="2\\^21"):
        r.align()
    # the VGICP-only calls refuse a plain GICP handle
    from gs_icp_slam_b200._lib import lib

    g = pygicp.FastGICP()
    assert lib.gsicp_vgicp_set_resolution(g._h, 1.0) == -4 and lib.gsicp_vgicp_voxel_count(g._h) == -4


def test_pickle_yields_fastvgicp(cuda):
    import pickle

    import pygicp

    r = pickle.loads(pickle.dumps(pygicp.FastVGICP()))
    assert type(r) is pygicp.FastVGICP
    assert r.get_voxel_mean_cov() == ([], [])


def test_fastgicp_unchanged_next_to_fastvgicp(cuda):
    import pygicp

    tgt, src, _ = S.gicp_pair(6000, 5000)

    def gicp_run():
        g = pygicp.FastGICP()
        g.set_max_correspondence_distance(0.05)
        g.set_max_knn_distance(99999)
        g.set_input_target(tgt)
        g.calculate_target_covariance_with_filter()
        g.set_input_source(src)
        g.set_source_filter(len(src), np.arange(1, len(src) + 1, dtype=np.int32))
        p = g.align()
        return p, g.get_final_hessian(), g.get_source_correspondence()

    before = gicp_run()
    v = _vgicp(tgt, src, 0.25, "DIRECT27")
    v.align()
    after = gicp_run()
    v.align()
    for a, b in zip(before[:2] + before[2], after[:2] + after[2]):
        assert np.array_equal(a, b)
