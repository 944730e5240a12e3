"""TEST INFRASTRUCTURE ONLY.  Pins the output side of neo360_b200.output (row f4) to the UNMODIFIED reference, imported through
oracle/ref_shim.py: `LitModel.psnr_each` (models/interface.py:53-61), `get_obj_rgbs_from_segmap` followed by `psnr_each`
(models/utils.py:102-109), the uint8 arrays `store_depth_img` hands to PIL (models/utils.py:29-43; captured by patching
`Image.fromarray`) and the text `write_stats` writes (models/utils.py:62-73).  Seeded frames with out-of-range values; masks that are
random, all zero and one pixel; depth sets that are random and constant (max = min).  Writes tests/golden/metrics_reference_vectors.npz.

    python oracle/make_golden_metrics.py        (CPU, this container only)
"""
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shim                     # noqa: E402

N, H, W, SEED = 4, 24, 32, 5

# results.json cases: (name, stat dicts in call order).  mip360 is the reference's Mip-NeRF 360 call (psnr, ssim, lpips, psnr_obj: two
# stats named "PSNR"); the numbers are arbitrary but typical.
STATS = {
    "neo360": [{"name": "PSNR", "mean": 23.456789012345, "test": 23.456789012345},
               {"name": "SSIM", "mean": 0.81234567890123, "test": 0.81234567890123},
               {"name": "LPIPS", "mean": 0.1234, "test": 0.1234}],
    "mip360": [{"name": "PSNR", "mean": 25.0, "test": 25.0},
               {"name": "SSIM", "mean": 0.9, "test": 0.9},
               {"name": "LPIPS", "mean": 0.2, "test": 0.2},
               {"name": "PSNR", "mean": 18.765432109876, "test": 18.765432109876}],
}


def inputs():
    g = torch.Generator().manual_seed(SEED)
    preds = 1.4 * torch.rand(N, H, W, 3, generator=g) - 0.2
    gts = 1.4 * torch.rand(N, H, W, 3, generator=g) - 0.2
    masks = torch.rand(N, H, W, generator=g) < 0.3
    masks[1] = False                 # empty mask: NaN
    masks[2] = False
    masks[2, 7, 11] = True           # one pixel
    depths = [2.0 + 3.0 * torch.rand(N, H, W, generator=g), torch.full((2, H, W), 1.75)]   # random; constant (max = min)
    return preds, gts, masks, depths


def main():
    ref_shim.load()
    import importlib
    utils = importlib.import_module("models.utils")
    LitModel = importlib.import_module("models.interface").LitModel
    preds, gts, masks, depths = inputs()
    psnr = LitModel.psnr_each(None, list(preds), list(gts))
    obj_p, obj_g = utils.get_obj_rgbs_from_segmap(list(masks), list(preds), list(gts))
    psnr_obj = LitModel.psnr_each(None, obj_p, obj_g)
    print("psnr", psnr.tolist(), "\npsnr_obj", psnr_obj.tolist())
    assert torch.isnan(psnr_obj[1]) and torch.isfinite(psnr_obj[[0, 2, 3]]).all()

    captured = {}
    orig = utils.Image.fromarray

    def grab(arr, *a, **k):
        captured.setdefault(cur, []).append(np.array(arr, copy=True))
        return orig(arr, *a, **k)

    utils.Image.fromarray = grab
    try:
        with tempfile.TemporaryDirectory() as d:
            for cur, ds in (("depth_rand", depths[0]), ("depth_const", depths[1])):
                utils.store_depth_img(d, list(ds), "depth_img")
            texts = {}
            for name, stats in STATS.items():
                path = os.path.join(d, f"{name}.json")
                utils.write_stats(path, *stats)
                with open(path, "rb") as f:
                    texts[name] = np.frombuffer(f.read(), dtype=np.uint8)
    finally:
        utils.Image.fromarray = orig
    out = os.path.join(ROOT, "tests", "golden", "metrics_reference_vectors.npz")
    np.savez_compressed(out, preds=preds.numpy(), gts=gts.numpy(), masks=masks.numpy(), psnr=psnr.numpy(), psnr_obj=psnr_obj.numpy(),
                        depth_rand=depths[0].numpy(), depth_const=depths[1].numpy(),
                        depth_img_rand=np.stack(captured["depth_rand"]), depth_img_const=np.stack(captured["depth_const"]),
                        **{f"stats_{k}": v for k, v in texts.items()})
    print("wrote", out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main()
