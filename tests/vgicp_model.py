"""float64 numpy restatement of fast_gicp's FastVGICP (FG/include/fast_gicp/gicp/fast_vgicp_voxel.hpp:129-160
create_voxelmap in ADDITIVE mode, fast_vgicp_impl.hpp:73-204 update_correspondences / linearize / compute_error), for the
VGICP tests.  The voxel sums run in point-index order (np.add.at), as the reference's append() sequence does, so the voxel
means are bit-identical to the reference's; voxels are listed in the CUDA map's order (packed key, 21 bits per axis)."""
import numpy as np

BITS = 21
# neighbor_offsets (fast_vgicp_voxel.hpp:10-44); DIRECT1 is the first entry of DIRECT7
OFFSETS7 = np.array([[0, 0, 0], [1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]], np.int64)
OFFSETS27 = np.array([[i - 1, j - 1, k - 1] for i in range(3) for j in range(3) for k in range(3)], np.int64)


def offsets(n):
    return {1: OFFSETS7[:1], 7: OFFSETS7, 27: OFFSETS27}[n]


def voxel_coord(x, res):
    """(x / res - 0.5).floor() per axis, as float64 (x: float64 or float32 points)."""
    return np.floor(np.asarray(x, np.float64) / res - 0.5)


def create_voxelmap(xyz, covs, res):
    """xyz (N, 3) float32 target points, covs (N, 3, 3) their covariances.  Returns dict(lo, dim, keys, count, mean (V, 3),
    cov (V, 3, 3)) with the voxels in ascending key order."""
    c = voxel_coord(np.asarray(xyz, np.float32), res).astype(np.int64)
    lo = c.min(0)
    dim = c.max(0) - lo + 1
    assert (dim <= (1 << BITS)).all(), "voxel extent needs more than 21 bits"
    r = c - lo
    key = r[:, 0] | (r[:, 1] << BITS) | (r[:, 2] << (2 * BITS))
    keys, inv, count = np.unique(key, return_inverse=True, return_counts=True)
    mean = np.zeros((len(keys), 3))
    cov = np.zeros((len(keys), 3, 3))
    np.add.at(mean, inv, np.asarray(xyz, np.float32).astype(np.float64))
    np.add.at(cov, inv, np.asarray(covs, np.float64))
    nd = count.astype(np.float64)
    return dict(lo=lo, dim=dim, keys=keys, count=count, mean=mean / nd[:, None], cov=cov / nd[:, None, None], res=res)


def transform(T, xyz):
    """Isometry3d * Vector4d (w = 1) in Eigen's evaluation order (rows 0-1 sequential, row 2 as a pairwise sum)."""
    T = np.asarray(T, np.float64)
    a = np.asarray(xyz, np.float32).astype(np.float64)
    x, y, z = a[:, 0], a[:, 1], a[:, 2]
    q0 = ((T[0, 0] * x + T[0, 1] * y) + T[0, 2] * z) + T[0, 3]
    q1 = ((T[1, 0] * x + T[1, 1] * y) + T[1, 2] * z) + T[1, 3]
    q2 = (T[2, 0] * x + T[2, 1] * y) + (T[2, 2] * z + T[2, 3])
    return np.stack([q0, q1, q2], 1)


def correspondences(vmap, src_xyz, src_covs, T, n_offsets):
    """(source index, voxel index, M) of every hit at pose T (fast_vgicp_impl.hpp:73-116)."""
    q = transform(T, src_xyz)
    c = voxel_coord(q, vmap["res"])
    src_i, vox_i = [], []
    for off in offsets(n_offsets):
        r = c + off - vmap["lo"]
        ok = np.all((r >= 0) & (r < vmap["dim"]), axis=1)
        ri = np.where(ok[:, None], r, 0).astype(np.int64)
        key = ri[:, 0] | (ri[:, 1] << BITS) | (ri[:, 2] << (2 * BITS))
        k = np.minimum(np.searchsorted(vmap["keys"], key), len(vmap["keys"]) - 1)
        hit = ok & (vmap["keys"][k] == key)
        src_i.append(np.nonzero(hit)[0])
        vox_i.append(k[hit])
    si, vi = np.concatenate(src_i), np.concatenate(vox_i)
    R = np.asarray(T, np.float64)[:3, :3]
    RCR = vmap["cov"][vi] + R @ np.asarray(src_covs, np.float64)[si] @ R.T
    return si, vi, np.linalg.inv(RCR)


def _skew(q):
    z = np.zeros(len(q))
    return np.stack([np.stack([z, -q[:, 2], q[:, 1]], 1), np.stack([q[:, 2], z, -q[:, 0]], 1),
                     np.stack([-q[:, 1], q[:, 0], z], 1)], 1)


def linearize(vmap, src_xyz, src_covs, T, n_offsets):
    """(H (6, 6), b (6,), error) at pose T (fast_vgicp_impl.hpp:118-180)."""
    si, vi, M = correspondences(vmap, src_xyz, src_covs, T, n_offsets)
    q = transform(T, src_xyz)[si]
    e = vmap["mean"][vi] - q
    w = np.sqrt(vmap["count"][vi].astype(np.float64))
    J = np.concatenate([_skew(q), -np.broadcast_to(np.eye(3), (len(q), 3, 3))], 2)  # (P, 3, 6)
    JtM = np.transpose(J, (0, 2, 1)) @ M
    H = np.einsum("p,pij->ij", w, JtM @ J)
    b = np.einsum("p,pi->i", w, (JtM @ e[:, :, None])[:, :, 0])
    err = float(np.sum(w * np.einsum("pi,pij,pj->p", e, M, e)))
    return H, b, err


def compute_error(vmap, src_xyz, src_covs, T0, Ti, n_offsets):
    """Error at Ti with the pairs and M of the linearisation pose T0 (fast_vgicp_impl.hpp:183-204)."""
    si, vi, M = correspondences(vmap, src_xyz, src_covs, T0, n_offsets)
    e = vmap["mean"][vi] - transform(Ti, src_xyz)[si]
    w = np.sqrt(vmap["count"][vi].astype(np.float64))
    return float(np.sum(w * np.einsum("pi,pij,pj->p", e, M, e)))


def as_reference_lists(vmap):
    """get_voxel_mean_cov's layout: (V, 4) means with w = 1 and (V, 4, 4) covariances with row / column 3 zero."""
    V = len(vmap["keys"])
    mean = np.concatenate([vmap["mean"], np.ones((V, 1))], 1)
    cov = np.zeros((V, 4, 4))
    cov[:, :3, :3] = vmap["cov"]
    return mean, cov


def sort_by_mean(mean, cov):
    """Voxels ordered by their mean (x, then y, then z): an order that does not depend on how a map lists them."""
    mean, cov = np.asarray(mean), np.asarray(cov)
    o = np.lexsort((mean[:, 2], mean[:, 1], mean[:, 0]))
    return mean[o], cov[o]
