"""Generates tests/golden/raster_ref_{cases,ext,full}.npz: golden records (tests/refgold.py) of the REFERENCE's own CUDA
code on the inputs of the rasterizer parity tests (tests/test_raster_gpu.py, tests/test_full_size_gpu.py) and of the simple-knn test
(tests/test_gicp_gpu.py).  Needs a GPU and the reference build of `make -C oracle ref` (oracle/_ref/libref_cuda.so and
the reference's torch extension under oracle/_ref/site):
    python tests/golden/make_raster_ref_cases_golden.py [OUT_DIR]"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)


def main(out_dir):
    import torch

    from oracle import ref_cuda, ref_ext
    from tests import refgold
    from tests import test_raster_gpu as T
    from tests.test_gicp_gpu import dist2_big_cloud
    from tests.util import scene_tensors

    cuda = torch.device("cuda:0")
    out = {}

    def add(name, arrays, extra_rows=()):
        out.setdefault(os.path.basename(T.gold_file(name)), {}).update(refgold.pack(name, arrays, extra_rows=extra_rows))
        print(name, {k: v.shape for k, v in arrays.items()}, flush=True)

    for P, size, degree, seed in T.FB_CASES:
        t, c, bg, gcol, gdep = T.case_fb(cuda, P, size, degree, seed)
        W, H = size
        add(f"fb_{P}_{degree}_{seed}", T.ref_outputs(T._ref(t, c, H, W, bg, degree), gcol, gdep))
    for active_degree, scale_modifier, size in T.OPTION_CASES:
        t, c, bg, gcol, gdep = T.case_options(cuda, active_degree, size)
        W, H = size
        ref = ref_cuda.RefRaster(bg, t["means3D"], t["shs"], None, t["opacities"].reshape(-1), t["scales"], t["rotations"], None,
                                 c["viewmatrix"], c["projmatrix"], c["campos"], c["tanfovx"], c["tanfovy"], H, W, active_degree,
                                 scale_modifier=scale_modifier)
        add(f"opt_{active_degree}", T.ref_outputs(ref, gcol, gdep))
    t, c, bg, gcol, gdep, a = T.case_degenerate(cuda)
    add("degenerate", T.ref_outputs(T._ref(t, c, 152, 200, bg), gcol, gdep), extra_rows=a.tolist())
    t, c, bg, colors, cov, gcol, gdep = T.case_precomputed(cuda)
    ref = ref_cuda.RefRaster(bg, t["means3D"], None, colors, t["opacities"].reshape(-1), None, None, cov, c["viewmatrix"],
                             c["projmatrix"], c["campos"], c["tanfovx"], c["tanfovy"], 240, 320, 0)
    add("precomputed", T.ref_outputs(ref, gcol, gdep))
    for P, lo, hi in T.CROWDED_CASES:
        t, c, bg = T.case_crowded(cuda, P)
        add(f"crowded_{P}", T.ref_outputs(T._ref(t, c, 120, 160, bg)))
    dgr = ref_ext.diff_gaussian_rasterization()
    for P, size, degree, seed in T.EXT_CASES:
        t, c, bg, gcol, gdep, active = T.case_ext(cuda, P, size, degree, seed)
        W, H = size
        depth, color, radii, is_used, g1, g2 = T.run_ext(dgr, t, c, H, W, bg, gcol, gdep, active)
        o = dict(radii=T._np(radii), is_used=T._np(is_used), depth=T._pix(depth), color=T._pix(color))
        o.update({"grad_" + k: T._np(g1[k]) for k in T.EXT_GRADS})
        add(f"ext_{P}_{degree}_{seed}", o)
    for P, size, scale in ((300000, (640, 480), 1.0), (1000000, (1280, 960), 2.0)):  # tests/test_full_size_gpu.py
        g, cm, t, c, cam = scene_tensors(P, 3 if P == 300000 else 4, cuda, size=size, scale=scale)
        W, H = size
        bg = torch.tensor([0.05, 0.1, 0.15], device=cuda)
        gen = torch.Generator(device="cpu").manual_seed(1)
        g1c = torch.randn((3, H, W), generator=gen).to(cuda)
        torch.randn((3, H, W), generator=gen)
        g1d = torch.randn((1, H, W), generator=gen).to(cuda)
        o = T.ref_outputs(T._ref(t, c, H, W, bg), g1c, g1d)
        del o["is_used"]
        add(f"full_{P}", o)
    add("dist2_200k", {"dist2": ref_cuda.ref_dist2(dist2_big_cloud(cuda)).cpu().numpy()})
    for f, arrays in out.items():
        path = os.path.join(out_dir, f)
        np.savez_compressed(path, **arrays)
        print(path, os.path.getsize(path))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden"))
