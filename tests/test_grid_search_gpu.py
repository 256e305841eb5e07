"""The grid neighbour search (gs_icp_slam_b200/csrc/grid.cuh) against brute force and the CPU oracle, bit for bit, on
clouds built to break it: points in the sliver between a cell face and where binning puts them (tests/grid_model.py),
degenerate and duplicated clouds, far outliers, queries outside the cloud, points exactly on cell faces — at the cloud
sizes that switch between the three grid builds (shared-memory, single-CTA, multi-kernel) and the two LM loops.

Every search entry point is reached: the single-query nearest neighbour (linearize), the multi-query one of the
persistent LM kernel (align), the k-NN of the covariances and distCUDA2's 3-NN.  The brute force runs on the GPU in
chunks with one torch op per rounding, ((dx*dx + dy*dy) + dz*dz) in float32, and ranks by (d2 bits << 32 | index):
the kernels' dist2_nofma and their lowest-index tie rule."""
import ctypes as C

import numpy as np
import pytest

from tests import grid_model as M

pytestmark = pytest.mark.gpu

SIZES = [25600, 25601, 65537]  # shared-memory build (<= 25 600 points), single-CTA build, multi-kernel build


def device_meta(handle, which=0):
    from gs_icp_slam_b200._lib import check, lib

    f, i = (C.c_float * 5)(), (C.c_int * 4)()
    check(lib.gsicp_test_grid_meta(handle, which, f, i), "gsicp_test_grid_meta")
    return tuple(int(v) for v in np.array(f[:], np.float32).view(np.uint32)), tuple(i[:])


def assert_same_geometry(meta, handle, which=0):
    """The model's grid is the device's, bit for bit; otherwise the adversarial cases test nothing."""
    assert device_meta(handle, which) == meta.as_tuple()


def brute_knn(cloud, queries, k, exclude_self=False, chunk=1024):
    """(d2 (m, k) float32, index (m, k) int64) of the k nearest cloud points of each query, on the GPU."""
    import torch

    dev = torch.device("cuda:0")
    p = torch.from_numpy(np.ascontiguousarray(cloud, np.float32)).to(dev)
    q = torch.from_numpy(np.ascontiguousarray(queries, np.float32)).to(dev)
    idx = torch.arange(p.shape[0], device=dev, dtype=torch.int64)
    out_d, out_i = [], []
    for s in range(0, q.shape[0], chunk):
        qq = q[s:s + chunk]
        dx = qq[:, None, 0] - p[None, :, 0]
        dy = qq[:, None, 1] - p[None, :, 1]
        dz = qq[:, None, 2] - p[None, :, 2]
        d2 = torch.add(torch.add(torch.mul(dx, dx), torch.mul(dy, dy)), torch.mul(dz, dz))
        key = (d2.view(torch.int32).to(torch.int64) << 32) | idx[None, :]
        if exclude_self:
            rows = torch.arange(qq.shape[0], device=dev)
            key[rows, rows + s] = torch.iinfo(torch.int64).max
        kk = torch.topk(key, k, dim=1, largest=False, sorted=True).values
        out_i.append((kk & 0xFFFFFFFF).cpu().numpy())
        out_d.append((kk >> 32).to(torch.int32).cpu().numpy().view(np.float32))
    return np.concatenate(out_d), np.concatenate(out_i)


def _regs(**kw):
    import pygicp
    from oracle import gicp_oracle as G

    regs = []
    for cls in (pygicp.FastGICP, G.FastGICP):
        r = cls()
        r.set_max_knn_distance(99999)
        for name, v in kw.items():
            getattr(r, name)(v)
        regs.append(r)
    return regs


def _dist2(points):
    import torch
    from simple_knn._C import distCUDA2

    return distCUDA2(torch.from_numpy(points).cuda()).cpu().numpy()


def _dist2_bruteforce(points):
    d, _ = brute_knn(points, points, 3, exclude_self=True)
    return ((d[:, 0] + d[:, 1]) + d[:, 2]) / np.float32(3)


# ---- face-sliver cases: one per search entry point -------------------------------------------------------------------
@pytest.mark.parametrize("n", SIZES)
def test_sliver_single_query_search(cuda, n):
    """linearize(identity): correspond_kernel -> grid_nn_warp."""
    cloud, meta, src, triples = M.sliver_cloud(n, 1, "nn", n_queries=3000)
    g, o = _regs()
    for r in (g, o):
        r.set_input_target(cloud)
        r.calculate_target_covariance()
        r.set_input_source(src)
        r.calculate_source_covariance()
        r.linearize(np.eye(4))
    assert_same_geometry(meta, g._h, 0)
    cg, dg = g.get_source_correspondence()
    co, do = o.get_source_correspondence()
    bd, bi = brute_knn(cloud, src, 1)
    assert [int(cg[t]) for t in range(len(triples))] == [p for p, _ in triples]
    assert np.array_equal(cg, bi[:, 0].astype(np.int32)) and np.array_equal(dg, bd[:, 0])
    assert np.array_equal(cg, co) and np.array_equal(dg, do)


@pytest.mark.parametrize("n", SIZES)
def test_sliver_multi_query_search(cuda, n):
    """align() with one iteration and <= 65 536 source points: align_lm_kernel -> grid_nn_warp_multi; the
    correspondences are those of the initial pose."""
    cloud, meta, src, triples = M.sliver_cloud(n, 1, "nn", n_queries=3000, seed=1)
    g, o = _regs(set_max_iterations=1)
    for r in (g, o):
        r.set_input_target(cloud)
        r.calculate_target_covariance()
        r.set_input_source(src)
        r.calculate_source_covariance()
        r.align(np.eye(4, dtype=np.float32))
    assert_same_geometry(meta, g._h, 0)
    cg, dg = g.get_source_correspondence()
    co, do = o.get_source_correspondence()
    bd, bi = brute_knn(cloud, src, 1)
    assert [int(cg[t]) for t in range(len(triples))] == [p for p, _ in triples]
    assert np.array_equal(cg, bi[:, 0].astype(np.int32)) and np.array_equal(dg, bd[:, 0])
    assert np.array_equal(cg, co) and np.array_equal(dg, do)


@pytest.mark.parametrize("k", [2, 20, 32])
@pytest.mark.parametrize("n", SIZES)
def test_sliver_covariance_knn(cuda, n, k):
    """calculate_target_covariance: knn_kernel -> grid_knn_warp, P deciding the k-th neighbour of each Q."""
    cloud, meta, q_idx, _ = M.sliver_cloud(n, k, "knn", seed=2)
    g, o = _regs(set_correspondence_randomness=k)
    for r in (g, o):
        r.set_input_target(cloud)
        r.calculate_target_covariance()
    assert_same_geometry(meta, g._h, 0)
    assert np.array_equal(g.get_target_rotationsq(), o.get_target_rotationsq())
    assert np.array_equal(g.get_target_scales(), o.get_target_scales())


@pytest.mark.parametrize("n", SIZES)
def test_sliver_dist2(cuda, n):
    """distCUDA2: dist2_kernel -> grid_knn_warp (k = 3, self excluded), with the old face rounded as one fma."""
    cloud, meta, q_idx, _ = M.sliver_cloud(n, 3, "dist2", fma=True, seed=3)
    out = _dist2(cloud)
    assert device_meta(None) == meta.as_tuple()
    ref = _dist2_bruteforce(cloud)
    assert np.array_equal(out[q_idx], ref[q_idx])
    assert np.array_equal(out, ref)


# ---- geometry sweep against brute force ---------------------------------------------------------------------------
KINDS = ["centred", "offset", "elongated", "planar", "collinear", "identical", "duplicated", "outlier", "clusters", "lattice"]


def sweep_cloud(kind, n, seed=0):
    """(cloud (n, 3) float32, queries (m, 3) float32): queries are jittered cloud points, points between and beyond."""
    rng = np.random.default_rng(seed)
    u = rng.uniform(-1, 1, size=(n, 3))
    if kind == "centred":
        c = u
    elif kind == "offset":
        c = u + 1000.0
    elif kind == "elongated":
        c = u * [50.0, 0.05, 0.05]
    elif kind == "planar":
        c = u * [1.0, 1.0, 0.0]
    elif kind == "collinear":
        c = u * [1.0, 0.0, 0.0] + [0.0, 3.0, -2.0]
    elif kind == "identical":
        c = np.zeros((n, 3)) + [0.25, -0.5, 2.0]
    elif kind == "duplicated":
        c = np.round(u * 4) / 4  # 9^3 distinct points, each repeated
    elif kind == "outlier":
        c = u * 0.5
        c[n // 2] = [1.0e4, -3.0e3, 2.0e3]
    elif kind == "clusters":
        c = u * 0.5
        c[: n // 2, 0] += 100.0
    elif kind == "lattice":  # points exactly on the faces of the grid this cloud gets
        corners = np.array([[-1, -1, -1], [1, 1, 1]], np.float32)
        meta = M.grid_choose(np.concatenate([corners, np.zeros((n - 2, 3), np.float32)]))
        ks = [rng.integers(0, int(d), size=n - 2) for d in meta.dims]
        body = np.stack([M.face(meta.o[d], ks[d], meta.cell) for d in range(3)], axis=1)
        c = np.concatenate([corners, body])
    c = np.asarray(c, np.float32) + np.float32(0)  # no -0.0: the device's fminf may keep either zero as the bbox minimum
    m = 2048
    lo, hi = c.min(0).astype(np.float64), c.max(0).astype(np.float64)
    span = np.maximum(hi - lo, 1e-3)
    pick = c[rng.integers(0, n, m)].astype(np.float64)
    jitter = pick + rng.normal(scale=1e-3, size=(m, 3)) * span
    between = lo + rng.uniform(0, 1, size=(m // 4, 3)) * span  # in the bounding box, e.g. between the clusters
    beyond = (lo + hi) / 2 + rng.uniform(-1.5, 1.5, size=(m // 4, 3)) * span  # half of them outside the bounding box
    q = np.concatenate([pick[: m // 4], jitter, between, beyond]).astype(np.float32)
    return c, q


@pytest.mark.parametrize("n", [25600, 25601, 65536, 65537])
@pytest.mark.parametrize("kind", KINDS)
def test_sweep_nearest_neighbour(cuda, kind, n):
    """linearize(identity) correspondences and squared distances against brute force, bit-exact."""
    cloud, q = sweep_cloud(kind, n)
    g, _ = _regs()
    g.set_input_target(cloud)
    g.calculate_target_covariance()
    g.set_input_source(q)
    g.calculate_source_covariance()
    g.linearize(np.eye(4))
    assert_same_geometry(M.grid_choose(cloud), g._h, 0)
    cg, dg = g.get_source_correspondence()
    bd, bi = brute_knn(cloud, q, 1)
    assert np.array_equal(cg, bi[:, 0].astype(np.int32))
    assert np.array_equal(dg, bd[:, 0])


@pytest.mark.parametrize("n", [25600, 25601, 65536, 65537])
@pytest.mark.parametrize("kind", KINDS)
def test_sweep_dist2(cuda, kind, n):
    """distCUDA2 (k = 3, self excluded) against brute force, bit-exact."""
    cloud, _ = sweep_cloud(kind, n, seed=1)
    out = _dist2(cloud)
    assert device_meta(None) == M.grid_choose(cloud).as_tuple()
    assert np.array_equal(out, _dist2_bruteforce(cloud))


@pytest.mark.parametrize("k", [2, 20, 32])
@pytest.mark.parametrize("kind", [k for k in KINDS if k != "identical"])  # identical: the oracle's kd-tree degenerates
def test_sweep_covariance_knn(cuda, kind, k):
    """k-NN of the covariances (65 537 points: multi-kernel build) against the oracle's exact kd-tree search."""
    cloud, _ = sweep_cloud(kind, 65537, seed=2)
    g, o = _regs(set_correspondence_randomness=k)
    for r in (g, o):
        r.set_input_target(cloud)
        r.calculate_target_covariance()
    assert_same_geometry(M.grid_choose(cloud), g._h, 0)
    assert np.array_equal(g.get_target_rotationsq(), o.get_target_rotationsq())
    assert np.array_equal(g.get_target_scales(), o.get_target_scales())


@pytest.mark.parametrize("n_src", [65536, 65537])
def test_align_source_size_switches_loop(cuda, n_src):
    """65 536 source points run the persistent LM kernel (grid_nn_warp_multi), 65 537 the host-driven loop
    (grid_nn_warp): both give the brute-force correspondences of the initial pose."""
    cloud, _ = sweep_cloud("centred", 25601, seed=3)
    src = sweep_cloud("centred", n_src, seed=4)[0] * np.float32(1.05)
    g, _ = _regs(set_max_iterations=1)
    g.set_input_target(cloud)
    g.calculate_target_covariance()
    g.set_input_source(src)
    g.calculate_source_covariance()
    g.align(np.eye(4, dtype=np.float32))
    cg, dg = g.get_source_correspondence()
    bd, bi = brute_knn(cloud, src, 1)
    assert np.array_equal(cg, bi[:, 0].astype(np.int32))
    assert np.array_equal(dg, bd[:, 0])
