"""TEST INFRASTRUCTURE ONLY -- NeO-360 golden vectors at 1 and 5 source views, minted from the UNMODIFIED reference.

    python oracle/make_golden_views.py        (CPU, where the reference tree exists)

NeO-360 is a few-view method: the reference's README renders and evaluates with 5 source views, and its test-time optimisation
takes 1, 3 or 5.  `oracle/make_golden.py` pins the oracle at NV = 3 only; this recipe runs its `e2e` unchanged at other view
counts and writes tests/golden/neo360_views_vectors.npz with the keys of the NV = 3 file (eval, train and randomized tuples, the
injected uniforms, the aux per-sample arrays), plus `<tag>_nv`.  The existing npz files are not touched.

`make_golden.e2e` builds its synthetic scene and the reference NeRF_TP with 3 views; here both constructors are wrapped so that they
receive the requested view count.  Everything else -- the rays, the reference calls, the oracle comparison at 5e-4 -- is `e2e`'s own.
The `src_imgs` it passes are read by the reference for their spatial size only (model.py:268-269; the encoder is bypassed).
"""
import contextlib
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import make_golden as mg  # noqa: E402
from oracle import ref_shim  # noqa: E402
from neo360_b200 import synth  # noqa: E402

# tag: (NV, img_wh, plane_hw, B, n_coarse, n_fine, seed).  The "small" case has B = 160 rays and N = 33 / 49 points per ray: B does not
# divide B * N evenly into views of N, so quirk Q1 conditions rows on rays of other pixels.
CASES = {
    "nv1_tiny": (1, (64, 48), (24, 32), 48, 16, 8, 0),
    "nv5_tiny": (5, (64, 48), (24, 32), 48, 16, 8, 0),
    "nv5_small": (5, (96, 64), (30, 40), 160, 32, 16, 1),
}


@contextlib.contextmanager
def views(nv):
    """Run make_golden's code with its scene and reference-module constructors fixed to `nv` source views."""
    saved = mg.synth, mg.ref_shim
    mg.synth = types.SimpleNamespace(**{k: getattr(synth, k) for k in dir(synth) if not k.startswith("__")})
    mg.synth.make_scene = lambda img_wh, _nv, plane_hw, seed: synth.make_scene(img_wh, nv, plane_hw, seed)
    mg.ref_shim = types.SimpleNamespace(**{k: getattr(ref_shim, k) for k in dir(ref_shim) if not k.startswith("__")})
    mg.ref_shim.make_reference_nerf_tp = lambda ns, nc, nf, _nv, seed: ref_shim.make_reference_nerf_tp(ns, nc, nf, nv, seed)
    try:
        yield
    finally:
        mg.synth, mg.ref_shim = saved


def main():
    ns = ref_shim.load()
    torch.set_grad_enabled(False)
    out = {}
    for tag, (nv, img_wh, plane_hw, B, nc, nf, seed) in CASES.items():
        with views(nv):
            mg.e2e(ns, out, tag, img_wh, plane_hw, B, nc, nf, seed)
        out[f"{tag}_nv"] = np.array(nv)
    path = os.path.join(mg.GOLD, "neo360_views_vectors.npz")
    np.savez_compressed(path, **{k: (v.numpy() if torch.is_tensor(v) else v) for k, v in out.items()})
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
