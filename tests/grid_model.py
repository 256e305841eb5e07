"""Float32 model of the device search grid (gs_icp_slam_b200/csrc/grid.cuh), for the grid search tests.

It restates, rounding for rounding:
- grid_choose: the cell size and the cell counts chosen from the bounding box and the point count;
- grid_cell_of: the cell a coordinate is binned into, under the old rule (a bare floor of (x - o) * inv_cell) and under
  the current one (that floor corrected by at most one cell against grid_face, so that face(i) <= x < face(i + 1));
- the cell face coordinate o + k * cell: two roundings (gicp.cu is compiled with -fmad=false, and grid_face rounds that
  way in every translation unit) or one fma (the old face of knn_dist2.cu, compiled with contraction on);
- ring_bound and the ring loop of grid_nn_warp / grid_knn_warp, so a query's result can be predicted under either rule.

`sliver_cloud` builds clouds with points placed in the sliver between a cell face and the place the old binning puts
it, each with a query whose search, under the old rule, stops one ring too early and returns a farther point.
"""
import numpy as np

f32 = np.float32
MAX_RING = 6
ONE_MINUS = f32(f32(1.0) - f32(1e-5))
EPS_CELL = f32(1e-6)


def max_cells(n):
    """DeviceGrid::build: cells allowed for a cloud of n points."""
    return int(min(max(2 * n, 4096), 1 << 24))


class Meta:
    def __init__(self, o, cell, inv_cell, dims):
        self.o = np.asarray(o, f32)
        self.cell = f32(cell)
        self.inv_cell = f32(inv_cell)
        self.dims = np.asarray(dims, np.int64)

    @property
    def ncells(self):
        return int(np.prod(self.dims))

    def as_tuple(self):
        """(ox, oy, oz, cell, inv_cell) as float32 bit patterns, (nx, ny, nz, ncells): the layout of gsicp_test_grid_meta."""
        f = np.array([*self.o, self.cell, self.inv_cell], f32).view(np.uint32)
        return tuple(int(v) for v in f), (*(int(d) for d in self.dims), self.ncells)


def grid_choose(pts):
    """grid_choose() on the NaN-ignoring bounding box of pts (n, 3) float32."""
    pts = np.asarray(pts, f32)
    n = pts.shape[0]
    lo, hi, ext = [], [], []
    for d in range(3):
        v = pts[:, d][~np.isnan(pts[:, d])]
        a, b = (f32(v.min()), f32(v.max())) if v.size else (f32(0), f32(0))
        if not b >= a:
            a = b = f32(0)
        lo.append(a)
        hi.append(b)
        ext.append(f32(b - a))
    emax = max(ext)
    e3 = f32(emax * f32(1e-3))
    vol = float(max(ext[0], e3)) * float(max(ext[1], e3)) * float(max(ext[2], e3))
    mc = max_cells(n)
    target = min(float(mc), max(64.0, 2.0 * n))
    cell = f32(np.cbrt(vol / target))
    if not cell > 0:
        cell = f32(1.0)
    dims = [1, 1, 1]
    for _ in range(64):
        dims = [int(min(f32(e / cell), f32(2.0e6))) + 1 for e in ext]
        if float(dims[0]) * dims[1] * dims[2] <= float(mc):
            break
        cell = f32(cell * f32(1.25))
    return Meta(lo, cell, f32(f32(1.0) / cell), dims)


def fma_f32(a, b, c):
    """Correctly rounded float32 a * b + c (a * b is exact in float64 for float32 inputs)."""
    a, b, c = (np.asarray(v, np.float64) for v in (a, b, c))
    p = a * b
    s = p + c
    # two-sum error of s, then break a float64 tie halfway between two float32s in the direction of the error
    bb = s - p
    err = (p - (s - bb)) + (c - bb)
    r = s.astype(f32)
    lo_ = np.nextafter(r, f32(-np.inf)).astype(np.float64)
    hi_ = np.nextafter(r, f32(np.inf)).astype(np.float64)
    mid = (s == (r.astype(np.float64) + lo_) / 2) | (s == (r.astype(np.float64) + hi_) / 2)
    nudged = np.where(err > 0, np.nextafter(s, np.inf), np.nextafter(s, -np.inf))
    return np.where(mid & (err != 0), nudged.astype(f32), r)


def face(o, k, cell, fma=False):
    """Coordinate of the lower face of cell k: o + k * cell, rounded twice (or once, as one fma)."""
    k = np.asarray(k, np.int64).astype(f32)
    if fma:
        return fma_f32(k, cell, o)
    return (f32(o) + (k * f32(cell)).astype(f32)).astype(f32)


def cell_of(meta, x, axis, fixed):
    """grid_cell_of along one axis (vectorised over x)."""
    x = np.asarray(x, f32)
    o, n = meta.o[axis], int(meta.dims[axis])
    with np.errstate(invalid="ignore"):
        c = np.floor(((x - o).astype(f32) * meta.inv_cell).astype(f32))
    c = np.nan_to_num(c, nan=0.0, posinf=2.0**31, neginf=-(2.0**31)).clip(0, n - 1).astype(np.int64)
    if fixed:
        below = x < face(o, c, meta.cell)
        above = x >= face(o, c + 1, meta.cell)
        c = np.where(below, np.maximum(c - 1, 0), np.where(above, np.minimum(c + 1, n - 1), c))
    return c


def cells_of(meta, pts, fixed):
    pts = np.asarray(pts, f32).reshape(-1, 3)
    return np.stack([cell_of(meta, pts[:, d], d, fixed) for d in range(3)], axis=1)


def dist2(p, q):
    """dist2_nofma: ((dx*dx + dy*dy) + dz*dz) in float32."""
    d = (np.asarray(p, f32) - np.asarray(q, f32)).astype(f32)
    sq = (d * d).astype(f32)
    return ((sq[..., 0] + sq[..., 1]).astype(f32) + sq[..., 2]).astype(f32)


def ring_lim(meta, c0, r, q, fixed, fma=False):
    """ring_bound: (lim, all).  The old rule's face is fma-rounded in the fma translation unit; the fixed one never is."""
    fm = fma and not fixed
    n = meta.dims
    allc = all(c0[d] - r <= 0 and c0[d] + r >= n[d] - 1 for d in range(3))
    bound = np.float32(np.finfo(f32).max)
    for d in range(3):
        if c0[d] - r > 0:
            bound = min(bound, f32(q[d] - face(meta.o[d], c0[d] - r, meta.cell, fm)))
        if c0[d] + r < n[d] - 1:
            bound = min(bound, f32(face(meta.o[d], c0[d] + r + 1, meta.cell, fm) - q[d]))
    safe = f32(f32(max(bound, f32(0)) * ONE_MINUS) - f32(EPS_CELL * meta.cell))
    return (f32(f32(safe * safe) * ONE_MINUS) if safe > 0 else f32(-1)), allc


def brute_knn(pts, q, k, exclude=-1):
    """k nearest of q in pts by (float32 d2, index)."""
    d = dist2(pts, q[None, :])
    idx = np.arange(pts.shape[0])
    keep = idx != exclude
    order = np.lexsort((idx[keep], d[keep]))[:k]
    return d[keep][order], idx[keep][order]


def search(meta, pts, q, k, fixed, exclude=-1, fma=False, first_ring=0, cells=None):
    """The ring loop of grid_knn_warp / grid_nn_warp (first_ring=1: grid_nn_warp_multi, which settles rings 0 and 1 as one
    block) under the old or the fixed rule: returns (d2, index) of the k results."""
    pts = np.asarray(pts, f32)
    q = np.asarray(q, f32)
    if cells is None:
        cells = cells_of(meta, pts, fixed)
    c0 = cells_of(meta, q, fixed)[0]
    cheb = np.abs(cells - c0[None, :]).max(axis=1)
    d = dist2(pts, q[None, :])
    idx = np.arange(pts.shape[0])
    want = min(k, pts.shape[0] - (1 if exclude >= 0 else 0))
    for r in range(first_ring, MAX_RING + 1):
        m = (cheb <= r) & (idx != exclude)
        order = np.lexsort((idx[m], d[m]))[:k]
        dk, ik = d[m][order], idx[m][order]
        lim, allc = ring_lim(meta, c0, r, q, fixed, fma)
        if allc or (lim > 0 and int((dk < lim).sum()) >= want):
            return dk, ik
    return brute_knn(pts, q, k, exclude)


def _sliver_faces(meta, fma, lo_cell, hi_cell):
    """Faces i along x (lo_cell <= i <= hi_cell) with the float32 x deepest below face(i) that the old rule bins into
    cell i, and those with the x deepest at or above face(i) binned into cell i - 1.  Returns [(i, x, side)] with side
    +1 for the first kind (the point lies below its cell) and -1 for the second, sorted by depth, deepest first."""
    i = np.arange(lo_cell, hi_cell + 1)
    fc = face(meta.o[0], i, meta.cell, fma)
    out = []
    for side in (+1, -1):
        x = fc.copy() if side < 0 else np.nextafter(fc, f32(-np.inf))
        best = np.full(i.shape, np.nan, f32)
        for _ in range(256):
            c = cell_of(meta, x, 0, False)
            hit = (c == i) if side > 0 else (c == i - 1)
            best = np.where(hit, x, best)
            x = np.nextafter(x, f32(-np.inf) if side > 0 else f32(np.inf)).astype(f32)
        ok = ~np.isnan(best)
        depth = np.abs(best.astype(np.float64) - fc.astype(np.float64)) / float(meta.cell)
        for j in np.flatnonzero(ok):
            out.append((int(i[j]), f32(best[j]), side, float(depth[j])))
    out.sort(key=lambda t: -t[3])
    return out


def sliver_cloud(n, k, mode, faces=6, half_extent=20.0, seed=0, fma=False, n_queries=0):
    """A cloud of exactly n points along x in [-half_extent, half_extent] (thin in y and z) with `faces` P/Q/R triples.

    For a triple at face i: P is binned by the old rule into the cell on the far side of face i; Q lies about 1.4 cells
    from the face on P's near side (so P is in the first ring Q's search has not reached when it stops); R lies beyond Q
    from P, a little farther than P but inside the old search's stopping radius.  A cluster of points close to Q makes P
    the k-th neighbour: k - 2 points when Q is itself a cloud point counted as its own neighbour (mode "knn"), k - 1 when
    it is excluded ("dist2"), none when the queries are separate points ("nn", k = 1).

    Returns (cloud (n, 3) float32, queries (m, 3) float32 for mode "nn" else the indices of the Q points in the cloud,
    list of (P index, R index) per triple).  The filler points lie in two blocks at the ends of the line, so they set
    the bounding box and do not come near any Q."""
    assert mode in ("nn", "knn", "dist2")
    rng = np.random.default_rng(seed)
    X = f32(half_extent)
    ext_yz = f32(2e-3)
    ends = np.array([[-X, 0, 0], [X, ext_yz, ext_yz]], f32)  # the bounding box corners
    n_cluster = {"nn": 0, "knn": k - 2, "dist2": k - 1}[mode]
    per = 2 + n_cluster + (0 if mode == "nn" else 1)
    n_fill = n - 2 - faces * per
    assert n_fill >= 0, "cloud too small for the requested triples"
    # the geometry depends only on the bounding box and n: fix both first
    meta = grid_choose(np.concatenate([ends, np.zeros((n - 2, 3), f32) + ends[0]]))
    nx = int(meta.dims[0])
    # triples in the middle third of the line, at least 12 cells apart
    cands = _sliver_faces(meta, fma, nx // 3, 2 * nx // 3)
    chosen, used = [], []
    y0, z0 = f32(1e-3), f32(1e-3)
    for i, px, side, _depth in cands:
        if len(chosen) == faces:
            break
        if any(abs(i - u) < 12 for u in used):
            continue
        fc = face(meta.o[0], i, meta.cell, fma)
        q = f32(fc - f32(side * 1.4) * meta.cell)
        qp = np.array([q, y0, z0], f32)
        pp = np.array([px, y0, z0], f32)
        dp = dist2(pp, qp)
        c0 = cells_of(meta, qp, False)[0]
        lim, _ = ring_lim(meta, c0, 1, qp, False, fma)
        if not (lim > dp):
            continue
        # R: on the other side of Q, strictly farther than P, strictly inside the stopping radius
        target = (np.sqrt(float(dp)) + np.sqrt(float(lim))) / 2
        rx = f32(q - f32(side * target))
        rp = np.array([rx, y0, z0], f32)
        dr = dist2(rp, qp)
        if not (dp < dr < lim):
            continue
        if not (cells_of(meta, rp, False)[0][0] in (c0[0] - 1, c0[0], c0[0] + 1)):
            continue
        chosen.append((qp, pp, rp))
        used.append(i)
    assert len(chosen) == faces, f"only {len(chosen)} usable sliver faces"
    pts = [ends]
    queries, triples, q_idx = [], [], []
    base = 2
    for qp, pp, rp in chosen:
        block = [pp, rp]
        if mode != "nn":
            block.append(qp)
        # cluster: within 0.05 cells of Q, spread a little in y and z, all nearer to Q than P is
        for _ in range(n_cluster):
            off = rng.uniform(-0.05, 0.05) * float(meta.cell)
            block.append(np.array([f32(qp[0] + f32(off)), f32(rng.uniform(0, float(ext_yz))), f32(rng.uniform(0, float(ext_yz)))], f32))
        triples.append((base, base + 1))
        if mode == "nn":
            queries.append(qp)
        else:
            q_idx.append(base + 2)
        pts.append(np.array(block, f32))
        base += len(block)
    # filler: two blocks of distinct points at the ends of the line, each 2 % of its length
    h = n_fill // 2
    fl = rng.uniform(0, 1, size=(n_fill, 3)).astype(f32)
    fx = np.where(np.arange(n_fill) < h, -X + f32(0.02 * 2 * X) * fl[:, 0], X - f32(0.02 * 2 * X) * fl[:, 0]).astype(f32)
    pts.append(np.stack([fx, fl[:, 1] * ext_yz, fl[:, 2] * ext_yz], axis=1).astype(f32))
    cloud = np.concatenate(pts).astype(f32)
    assert cloud.shape[0] == n
    chk = grid_choose(cloud)
    assert chk.as_tuple() == meta.as_tuple(), "the triples moved the bounding box"
    if mode == "nn":
        q = np.array(queries, f32)
        if n_queries > len(q):  # extra queries spread over the line, so the source has a 3-D extent of its own
            extra = np.stack([rng.uniform(-float(X), float(X), n_queries - len(q)), rng.uniform(0, float(ext_yz), n_queries - len(q)),
                              rng.uniform(0, float(ext_yz), n_queries - len(q))], axis=1).astype(f32)
            q = np.concatenate([q, extra])
        return cloud, meta, q, triples
    return cloud, meta, np.array(q_idx), triples
