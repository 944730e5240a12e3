"""oracle/pixelnerf_oracle.py reproduces the unmodified reference PixelNeRF (tests/golden/pixelnerf_reference_vectors.npz, minted by
oracle/make_golden_pixelnerf.py): stage tensors and both levels' outputs, deterministic with white_bkgd and randomized (injected uniforms)
without, NV 1 and 3, caller chunks of 8 and 1024 rays (quirk Q1), near / far honoured and view-0 intrinsics."""
import os

import numpy as np
import pytest
import torch

from neo360_b200 import synth
from oracle import pixelnerf_oracle as por

GOLD = os.path.join(os.path.dirname(__file__), "golden", "pixelnerf_reference_vectors.npz")
TAGS = ("p1_b8", "p3_b8", "p3_b1024")
NEAR, FAR = 0.02, 3.0


def case(z, tag):
    W, H, nv, B, nc, nf, seed = (int(x) for x in z[f"{tag}_cfg"])
    g = lambda k: torch.from_numpy(z[f"{tag}_{k}"])
    sc = synth.make_scene((W, H), nv, (8, 8), seed)
    osc = por.scene(sc["latent"], sc["src_poses"], g("src_focal"), g("src_c"), (W, H))
    rays = {k: g(k) for k in ("rays_o", "rays_d", "viewdirs")}
    return osc, rays, synth.make_pixelnerf_params(seed), (nc, nf), {"u0": g("u0"), "u1": g("u1")}


@pytest.mark.parametrize("tag", TAGS)
def test_outputs_match_reference(tag):
    z = np.load(GOLD)
    osc, rays, P, (nc, nf), rnd = case(z, tag)
    with torch.no_grad():
        ev = por.render(rays, osc, P, nc, nf, NEAR, FAR, True)
        rr = por.render(rays, osc, P, nc, nf, NEAR, FAR, False, rand=rnd)
    for lvl in range(2):
        for i, name in enumerate(("rgb", "acc", "depth")):
            for got, mode in ((ev, "eval"), (rr, "rand")):
                ref = torch.from_numpy(z[f"{tag}_{mode}{lvl}_{name}"])
                assert float((got[lvl][i] - ref).abs().max()) < 2e-5, (tag, mode, lvl, name)


@pytest.mark.parametrize("tag", ("p1_b8", "p3_b8"))
def test_stages_match_reference(tag):
    z = np.load(GOLD)
    osc, rays, _, _, _ = case(z, tag)
    t = torch.linspace(0.0, 1.0, 6)
    t = NEAR * (1.0 - t) + FAR * t
    pts = rays["rays_o"][:, None, :] + t[None, :, None] * rays["rays_d"][:, None, :]
    st = por.stages(pts, rays["viewdirs"], osc, 6)
    ref = lambda k: torch.from_numpy(z[f"{tag}_stage_{k}"])
    assert float((st["p_cam"] - ref("cam")).abs().max()) < 1e-6
    assert float((st["uv"] - ref("uv")).abs().max()) < 1e-3           # pixels
    assert float((st["latent"] - ref("latent")).abs().max()) < 1e-5
    assert float((st["dir_tile"] - ref("dir_tile")).abs().max()) < 1e-6


def test_fixture_exercises_quirks():
    """The fixture's per-view intrinsics differ (only view 0 may be used) and the two chunk sizes give different Q1 conditioning."""
    z = np.load(GOLD)
    f, c = z["p3_b8_src_focal"], z["p3_b8_src_c"]
    assert f[1] != f[0] and (c[1] != c[0]).all()
    osc, rays, P, (nc, nf), _ = case(z, "p3_b1024")
    with torch.no_grad():
        whole = por.render(rays, osc, P, nc, nf, NEAR, FAR, True)[1][0]
        part = por.render({k: v[:8] for k, v in rays.items()}, osc, P, nc, nf, NEAR, FAR, True)[1][0]
    assert float((whole[:8] - part).abs().max()) > 1e-4
