"""Generates tests/golden/raster_ref_small.npz from the REFERENCE's own CUDA rasterizer (oracle/_ref/libref_cuda.so,
built unmodified from the reference's sources by `make -C oracle ref`).  Needs a GPU:
    python tests/golden/make_raster_golden.py
The fixture pins oracle/raster_oracle.c (tests/test_raster_oracle.py, CPU) and the CUDA path (tests/test_raster_gpu.py)
to outputs of the reference itself: colour, depth, radii, is_used, num_rendered, sorted point_list, ranges, 8 gradients."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import ref_cuda  # noqa: E402
from tests.util import scene_tensors  # noqa: E402

CASES = [dict(name="deg1", P=6000, seed=11, size=(96, 64), degree=1, bg=(0.0, 0.5, 1.0)),
         dict(name="deg0", P=12000, seed=12, size=(128, 80), degree=0, bg=(0.1, 0.2, 0.3))]


def main():
    dev = torch.device("cuda:0")
    out = {}
    for cs in CASES:
        W, H = cs["size"]
        g, cm, t, c, cam = scene_tensors(cs["P"], cs["seed"], dev, sh_degree=cs["degree"], size=cs["size"])
        bg = torch.tensor(cs["bg"], device=dev)
        ref = ref_cuda.RefRaster(bg, t["means3D"], t["shs"], None, t["opacities"].reshape(-1), t["scales"], t["rotations"], None,
                                 c["viewmatrix"], c["projmatrix"], c["campos"], c["tanfovx"], c["tanfovy"], H, W, cs["degree"])
        rng = np.random.default_rng(cs["seed"] + 100)
        # upstream gradients are stored as float16 in the fixture: round them BEFORE running the reference
        gcol = rng.normal(size=(3, H, W)).astype(np.float16).astype(np.float32)
        gdep = rng.normal(size=(1, H, W)).astype(np.float16).astype(np.float32)
        pl, rg = ref.export()
        grads = ref.backward(torch.from_numpy(gcol).to(dev), torch.from_numpy(gdep).to(dev))
        n = cs["name"]
        out[f"{n}_color"], out[f"{n}_depth"] = ref.color.cpu().numpy(), ref.depth.cpu().numpy()
        out[f"{n}_radii"], out[f"{n}_is_used"] = ref.radii.cpu().numpy(), ref.is_used.cpu().numpy()
        out[f"{n}_num_rendered"] = np.int64(ref.num_rendered)
        out[f"{n}_point_list"], out[f"{n}_ranges"] = pl.cpu().numpy().astype(np.int32), rg.cpu().numpy().astype(np.int32)
        out[f"{n}_gcol"], out[f"{n}_gdep"] = gcol.astype(np.float16), gdep.astype(np.float16)
        for k in ("means2D", "colors", "opacity", "means3D", "cov3D", "sh", "scales", "rotations"):
            out[f"{n}_grad_{k}"] = grads[k].cpu().numpy()
        ref.free()
        print(n, "R =", ref.num_rendered, "V =", int((out[f"{n}_radii"] > 0).sum()))
    np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), "raster_ref_small.npz"), **out)


if __name__ == "__main__":
    main()
