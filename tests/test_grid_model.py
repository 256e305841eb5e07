"""The float32 grid model (tests/grid_model.py) and its adversarial clouds, on the CPU: the face-sliver triples are misses
under the old binning rule and hits under the current one, so the GPU tests built on them test something."""
import numpy as np
import pytest

from tests import grid_model as M


def test_face_helpers():
    meta = M.grid_choose(np.array([[-20, 0, 0], [20, 2e-3, 2e-3]] + [[0, 0, 0]] * 49999, np.float32))
    assert tuple(meta.dims) == (4642, 1, 1) and abs(meta.cell - 0.0086177) < 1e-7  # the line cloud of the issue's example
    k = np.arange(0, 4643)
    # the face is monotone and the fma rounding differs from the two-rounding one at some faces
    for fma in (False, True):
        f = M.face(meta.o[0], k, meta.cell, fma)
        assert (np.diff(f.astype(np.float64)) > 0).all()
    assert (M.face(meta.o[0], k, meta.cell, True) != M.face(meta.o[0], k, meta.cell, False)).any()
    # fixed binning: face(i) <= x < face(i + 1) for every float32 near the faces
    x = np.concatenate([np.nextafter(M.face(meta.o[0], k, meta.cell), np.float32(s * np.inf)) for s in (-1, 1)] +
                       [M.face(meta.o[0], k, meta.cell)]).astype(np.float32)
    x = x[(x >= meta.o[0]) & (x <= np.float32(20))]
    c = M.cell_of(meta, x, 0, fixed=True)
    inner = c < 4641
    assert (x >= M.face(meta.o[0], c, meta.cell)).all()
    assert (x[inner] < M.face(meta.o[0], c[inner] + 1, meta.cell)).all()
    # ... which the old rule violates
    c_old = M.cell_of(meta, x, 0, fixed=False)
    assert (c_old != c).any()


def test_fma_f32_is_correctly_rounded():
    rng = np.random.default_rng(1)
    a, b, c = (rng.normal(size=20000).astype(np.float32) for _ in range(3))
    from fractions import Fraction

    got = M.fma_f32(a, b, c)
    for i in range(0, 20000, 97):
        exact = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        r = np.float32(got[i])
        lo, hi = np.nextafter(r, np.float32(-np.inf)), np.nextafter(r, np.float32(np.inf))
        err = abs(Fraction(float(r)) - exact)
        assert err <= abs(Fraction(float(lo)) - exact) and err <= abs(Fraction(float(hi)) - exact)


@pytest.mark.parametrize("mode,k,fma,first_ring", [("nn", 1, False, 0), ("nn", 1, False, 1), ("knn", 2, False, 0),
                                                   ("knn", 20, False, 0), ("knn", 32, False, 0), ("dist2", 3, True, 0)])
@pytest.mark.parametrize("n", [25600, 25601, 65537])
def test_sliver_triples_miss_under_old_rule_and_hit_under_fixed_rule(mode, k, fma, first_ring, n):
    cloud, meta, queries, triples = M.sliver_cloud(n, k, mode, fma=fma)
    assert tuple(meta.dims[1:]) == (1, 1) and meta.dims[0] > 1000
    cells = {fixed: M.cells_of(meta, cloud, fixed) for fixed in (False, True)}
    for t, (p, r) in enumerate(triples):
        if mode == "nn":
            q, excl = queries[t], -1
        else:
            q, excl = cloud[queries[t]], (queries[t] if mode == "dist2" else -1)
        bd, bi = M.brute_knn(cloud, q, k, excl)
        assert bi[k - 1] == p  # P is the k-th neighbour
        od, oi = M.search(meta, cloud, q, k, False, excl, fma, first_ring, cells[False])
        assert oi[k - 1] == r and od[k - 1] > bd[k - 1]  # the old rule stops early and returns R instead
        nd, ni = M.search(meta, cloud, q, k, True, excl, fma, first_ring, cells[True])
        assert np.array_equal(ni, bi) and np.array_equal(nd, bd)
