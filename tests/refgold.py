"""Compact golden records of the reference's outputs, so that the parity tests run without the reference build.

A record stores, for every array of a reference run: its shape, dtype and SHA-256 of its bytes (bit-exact comparisons keep
their full strength).  For the comparisons that allow round-off it also stores, for float arrays: the SHA-256 of the mask
of finite elements, the largest finite |value|, a fixed, seeded sample of rows (the rows with the largest |value| among
them), and over BLOCKS contiguous blocks of rows the largest |value| and the sums of the values and of their magnitudes,
so that every row takes part in the comparison.  Records are written by tests/golden/make_*.py."""
import hashlib

import numpy as np

SAMPLE_ROWS = 256
TOP_ROWS = 32
BLOCKS = 256


def _rows(a):
    a = np.asarray(a)
    return a.reshape(a.shape[0] if a.ndim > 1 else a.size, -1) if a.size else a.reshape(0, 1)


def _edges(n):
    return np.linspace(0, n, min(n, BLOCKS) + 1).astype(np.int64)


def _block_stats(r):
    """Per block of rows: largest finite |value|, sum of the finite values, sum of their magnitudes (float64)."""
    f = np.where(np.isfinite(r), r, 0.0).astype(np.float64)
    e = _edges(r.shape[0])
    mx = np.array([np.abs(f[a:b]).max() for a, b in zip(e[:-1], e[1:])])
    return mx, np.add.reduceat(f.sum(1), e[:-1]), np.add.reduceat(np.abs(f).sum(1), e[:-1]), np.diff(e) * r.shape[1]


def _sha(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8)


def pack(prefix, arrays, extra_rows=(), seed=0, sample=True):
    """{f"{prefix}.{name}.{field}": ndarray} for np.savez: see the module docstring.  sample=False keeps only what the
    bit-exact comparisons need."""
    out = {}
    for name, a in arrays.items():
        a = np.asarray(a)
        k = f"{prefix}.{name}"
        out[k + ".shape"] = np.array(a.shape, np.int64)
        out[k + ".dtype"] = np.array(a.dtype.str)
        out[k + ".sha"] = _sha(a)
        if sample and a.dtype.kind == "f" and a.size:
            r = _rows(a)
            fin = np.where(np.isfinite(r), np.abs(r), 0.0)
            n = r.shape[0]
            rng = np.random.default_rng(seed)
            idx = set(rng.choice(n, size=min(n, SAMPLE_ROWS), replace=False).tolist())
            idx |= set(np.argsort(fin.max(1))[-TOP_ROWS:].tolist())
            idx |= {int(i) for i in extra_rows if 0 <= int(i) < n}
            idx = np.array(sorted(idx), np.int64)
            out[k + ".idx"], out[k + ".val"] = idx, r[idx]
            out[k + ".absmax"] = np.array(fin.max(), np.float64)
            out[k + ".finite"] = _sha(np.isfinite(a))
            out[k + ".bmax"], out[k + ".bsum"], out[k + ".babs"], _ = _block_stats(r)
        if a.size <= 64:
            out[k + ".full"] = a
    return out


class Record:
    """One golden record (the `prefix` of pack) loaded from an .npz file."""

    def __init__(self, path, prefix):
        self.g, self.p = np.load(path), prefix

    def __contains__(self, name):
        return f"{self.p}.{name}.sha" in self.g.files

    def _get(self, name, field):
        return self.g[f"{self.p}.{name}.{field}"]

    def _meta(self, name, a):
        a = np.asarray(a)
        assert tuple(a.shape) == tuple(self._get(name, "shape")), (name, a.shape, tuple(self._get(name, "shape")))
        assert a.dtype.str == str(self._get(name, "dtype")), (name, a.dtype.str, str(self._get(name, "dtype")))
        return a

    def full(self, name):
        """The reference's array itself (kept for arrays of at most 64 elements)."""
        return self.g[f"{self.p}.{name}.full"]

    def same(self, name, a):
        """True when `a` is bit-identical to the reference's array."""
        a = self._meta(name, a)
        return np.array_equal(_sha(a), self._get(name, "sha"))

    def exact(self, name, a):
        assert self.same(name, a), f"{name}: not bit-identical to the reference"

    def sample(self, name, a):
        """(sampled row indices, our rows there, the reference's rows there, the reference's largest finite |value|)."""
        a = self._meta(name, a)
        idx = self._get(name, "idx")
        return idx, _rows(a)[idx], self._get(name, "val"), float(self._get(name, "absmax"))

    def finite_matches(self, name, a):
        """True when `a` is finite exactly where the reference's array is."""
        a = self._meta(name, a)
        return np.array_equal(_sha(np.isfinite(a)), self._get(name, "finite"))

    def rel_err(self, name, a):
        """tests.util.rel_err (max |a-b| / max |b|) from what the record holds: inf unless `a` is finite exactly where the
        reference is; otherwise the largest of the lower bounds on max |a-b| that the record gives — the sampled rows
        exactly, and over every row: the difference of the largest |value|s of the whole array and of each block, and each
        block's difference of sums (and of sums of magnitudes) divided by its element count — over max |b|."""
        if self.same(name, a):
            return 0.0
        if not self.finite_matches(name, a):
            return float("inf")
        _, x, y, m = self.sample(name, a)
        fin = np.isfinite(y)
        d = [np.where(fin, np.abs(x.astype(np.float64) - np.where(fin, y, 0.0)), 0.0).max() if x.size else 0.0]
        r = _rows(a)
        if r.size:
            mx, sm, ab, cnt = _block_stats(r)
            d.append(abs(float(mx.max()) - m))
            d.append(float(np.abs(mx - self._get(name, "bmax")).max()))
            d.append(float((np.abs(sm - self._get(name, "bsum")) / cnt).max()))
            d.append(float((np.abs(ab - self._get(name, "babs")) / cnt).max()))
        return float(max(d) / (m + 1e-30))


# Replay of the reference's vendored Eigen (oracle/gicp_eigen_ref.cpp) for tests/test_gicp_oracle.py: every call's outputs,
# in call order, recorded by tests/golden/make_reference_cpu_golden.py.  Per function: the arguments as (role, count, ctype);
# role "in" is a pointer input (its sum is recorded and checked, so a replay out of step fails), "out" a pointer output,
# "int" a scalar, "ref" a c_double passed by reference.
EIGEN_SIGNATURES = {
    "eig_svd3": (("in", 9, "d"), ("out", 9, "d"), ("out", 3, "d"), ("out", 9, "d")),
    "eig_quat_from_matrix": (("in", 9, "d"), ("out", 4, "d")),
    "eig_cov_pipeline": (("in", 9, "d"), ("int", 1, "i"), ("out", 4, "f"), ("out", 3, "f"), ("out", 9, "d")),
    "eig_cov_from_qs": (("in", 4, "f"), ("in", 3, "f"), ("out", 9, "d")),
    "eig_mahalanobis": (("in", 9, "d"), ("in", 9, "d"), ("in", 16, "d"), ("out", 9, "d")),
    "eig_linearize_point": (("in", 16, "d"), ("in", 3, "f"), ("in", 3, "f"), ("in", 9, "d"), ("out", 36, "d"), ("out", 6, "d"),
                            ("ref", 1, "d")),
    "eig_ldlt_solve6": (("in", 36, "d"), ("in", 6, "d"), ("out", 6, "d")),
    "eig_so3_exp": (("in", 3, "d"), ("out", 9, "d")),
}


def _view(arg, count, code):
    import ctypes as C

    arg = getattr(arg, "_obj", arg)  # ctypes.byref(x) -> x
    if isinstance(arg, C.c_double):
        return np.ctypeslib.as_array((C.c_double * 1).from_address(C.addressof(arg)))
    ptr = arg.value if isinstance(arg, C.c_void_p) else arg
    t = C.c_double if code == "d" else C.c_float
    return np.ctypeslib.as_array((t * count).from_address(ptr))


class EigenRecorder:
    """Wraps the real library: forwards every call and records its input sums and outputs."""

    def __init__(self, lib):
        self.lib, self.calls = lib, {n: [] for n in EIGEN_SIGNATURES}

    def __getattr__(self, name):
        sig, fn = EIGEN_SIGNATURES[name], getattr(self.lib, name)

        def call(*args):
            ins = [float(_view(a, n, c).astype(np.float64).sum()) for a, (r, n, c) in zip(args, sig) if r == "in"]
            fn(*args)
            outs = [_view(a, n, c).copy() for a, (r, n, c) in zip(args, sig) if r in ("out", "ref")]
            self.calls[name].append((ins, outs))

        return call

    def arrays(self, prefix):
        out = {}
        for name, calls in self.calls.items():
            if calls:
                out[f"{prefix}.{name}.in"] = np.array([c[0] for c in calls], np.float64)
                for j in range(len(calls[0][1])):
                    out[f"{prefix}.{name}.out{j}"] = np.stack([c[1][j] for c in calls])
        return out


class EigenReplay:
    """Stands in for the library: each call checks its input sums and writes the recorded outputs."""

    def __init__(self, path, prefix):
        self.g, self.p, self.pos = np.load(path), prefix, {}

    def __getattr__(self, name):
        sig = EIGEN_SIGNATURES[name]

        def call(*args):
            k = self.pos.get(name, 0)
            self.pos[name] = k + 1
            ins = [float(_view(a, n, c).astype(np.float64).sum()) for a, (r, n, c) in zip(args, sig) if r == "in"]
            rec = self.g[f"{self.p}.{name}.in"]
            assert k < len(rec), f"{name}: more calls than recorded"
            assert np.allclose(ins, rec[k], rtol=1e-12, atol=0), f"{name} call {k}: inputs differ from the recorded run"
            j = 0
            for a, (r, n, c) in zip(args, sig):
                if r in ("out", "ref"):
                    _view(a, n, c)[:] = self.g[f"{self.p}.{name}.out{j}"][k]
                    j += 1

        return call
