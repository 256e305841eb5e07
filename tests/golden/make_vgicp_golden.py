"""Generates tests/golden/vgicp_ref_cases.npz: the REFERENCE's own FastVGICP (fast_gicp's unmodified fast_vgicp.cpp and
pybind11 module, oracle/_ref/fast_gicp built by `make -C oracle ref` where the reference's sources are present) on every case of
tests/vgicp_cases.py, as golden records (tests/refgold.py).  Every case with a pose is run with 1 OpenMP thread and with
all threads; the two poses must agree to 1e-7.  Run in the build container:
    python tests/golden/make_vgicp_golden.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)


def main():
    from oracle import ref_gicp
    from tests import refgold
    from tests import vgicp_cases as cases

    m = ref_gicp.load()

    def factory(threads):
        def make():
            r = m.FastVGICP()
            if threads:
                r.set_num_threads(threads)
            return r

        return make

    out = {}
    for name, (fn, kw, posed) in cases.CASES.items():
        a = fn(factory(0), **kw)
        if posed:
            b = fn(factory(1), **kw)
            for k in a:
                if k.startswith("pose"):
                    d = np.abs(a[k].astype(np.float64) - b[k]).max()
                    assert d <= 1e-7, (name, k, d)
        arrays = {k: v for k, v in a.items() if posed or not k.startswith(("pose", "H"))}
        for k, v in arrays.items():
            out.update(refgold.pack(name, {k: v}, sample=not k.startswith("vmean")))
        print(name, {k: v.shape for k, v in arrays.items()}, flush=True)
    path = os.path.join(ROOT, "tests", "golden", "vgicp_ref_cases.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path))


if __name__ == "__main__":
    main()
