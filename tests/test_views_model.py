"""CPU: NeO-360 at 1 and 5 source views and the test-time optimisation recipe.

* the oracle against golden vectors minted from the UNMODIFIED reference at NV = 1 and 5 (oracle/make_golden_views.py);
* the host draws of a test-time optimisation sample against the reference dataset's statements (nerds360_ae.py:540-551, 598-673);
* the optimiser the recipe builds (model.py:957-981)."""
import os
import random

import numpy as np
import pytest
import torch

from neo360_b200 import batches, synth, training
from oracle import neo360_oracle as orc

T = lambda a: torch.from_numpy(np.asarray(a))
TAGS = ["nv1_tiny", "nv5_tiny", "nv5_small"]
EV = ("comp_rgb", "fg_rgb", "bg_rgb", "fg_acc", "bg_lambda", "depth")
TR = ("comp_rgb", "fg_w", "bg_w", "fg_sdist", "bg_sdist", "bg_acc")


@pytest.fixture(scope="module")
def vgolden():
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "neo360_views_vectors.npz"))


def load_case(g, tag):
    """The synthetic scene, weights and rays of one case (the scene is regenerated from its seed and checked against the stored
    checksum)."""
    W, H, hp, wp, B, nc, nf, seed, start = [int(x) for x in g[f"{tag}_cfg"]]
    nv = int(g[f"{tag}_nv"])
    sc = synth.make_scene((W, H), nv, (hp, wp), seed)
    chk = np.array([float(sc[k].double().sum()) for k in ("planes_xz", "planes_xy", "planes_yz", "latent")]
                   + [float(sc[k].double().abs().sum()) for k in ("planes_xz", "latent")])
    assert np.allclose(chk, g[f"{tag}_checksum"], rtol=1e-9), "synthetic scene RNG drifted; re-mint the goldens"
    rays = {k: T(g[f"{tag}_{k}"]) for k in ("rays_o", "rays_d", "viewdirs")}
    return nv, sc, synth.make_mlp_params(seed), rays, (W, H, nc, nf)


@pytest.mark.parametrize("tag", TAGS)
def test_oracle_vs_reference_vectors(vgolden, tag):
    g = vgolden
    nv, sc, P, rays, (W, H, nc, nf) = load_case(g, tag)
    assert sc["src_poses"].shape[0] == nv and g[f"{tag}_aux0_fg_sigma"].shape[0] == rays["rays_o"].shape[0]
    osc = orc.Scene(sc["planes_xz"], sc["planes_xy"], sc["planes_yz"], sc["latent"], sc["src_poses"],
                    float(sc["src_focal"][0]), float(sc["src_c"][0, 0]), float(sc["src_c"][0, 1]), W, H)
    with torch.no_grad():
        ev, aux = orc.render(rays, osc, P, nc, nf, False, True, return_aux=True)
        tr = orc.render(rays, osc, P, nc, nf, True, False)
        rr = orc.render(rays, osc, P, nc, nf, False, True, rand={k: T(g[f"{tag}_u_{k}"]) for k in ("fg0", "bg0", "fg1", "bg1")})
    tol = 5e-4      # the oracle's pin tolerance (oracle/make_golden.py)
    for lvl in range(2):
        for names, got, kind in ((EV, ev, "eval"), (TR, tr, "train"), (EV, rr, "rand")):
            for n, v in zip(names, got[lvl]):
                assert float((v - T(g[f"{tag}_{kind}{lvl}_{n}"])).abs().max()) < tol, (kind, lvl, n)
        for k in ("fg_sigma", "bg_sigma", "fg_rgb", "bg_rgb"):
            assert float((aux[lvl][k] - T(g[f"{tag}_aux{lvl}_{k}"])).abs().max()) < tol, (lvl, k)


def reference_draws(src_views_num, H, W, patch, ray_batch_size=500):
    """The statements of the reference dataset's --is_optimize sample (nerds360_ae.py:550, 638-664, 666-667), verbatim."""
    dest_view_num = random.sample(src_views_num, 1)[0]
    if patch:
        x = np.random.randint(0, H - 30 + 1)
        y = np.random.randint(0, W - 30 + 1)
        return dest_view_num, (x, y)
    return dest_view_num, torch.randint(0, H * W, (ray_batch_size,))


@pytest.mark.parametrize("ids", [[0], [0, 38, 44], [0, 38, 44, 94, 48]], ids=["1", "3", "5"])
@pytest.mark.parametrize("patch", [False, True], ids=["rays", "patch"])
def test_source_view_draws_follow_the_reference(ids, patch):
    """Ten successive samples under the same `random`, numpy and torch seeds: the same view position, pixels and patch origins."""
    H, W = 48, 64
    seed = 7

    def seq(fn):
        random.seed(seed)
        np.random.seed(seed)
        torch.manual_seed(seed)
        return [fn() for _ in range(10)]

    ref = seq(lambda: reference_draws(ids, H, W, patch))
    got = seq(lambda: batches.draw_source_view(len(ids), H, W, finetune_lpips=patch))
    assert len(ids) == 1 or len({r[0] for r in ref}) > 1                          # the draws do move between views
    for (rv, rd), (v, d) in zip(ref, got):
        assert ids[v] == rv
        if patch:
            assert d == tuple(int(t) for t in rd)
        else:
            assert torch.equal(d, v * H * W + rd)


def test_source_view_draws_with_a_generator_and_a_fixed_view():
    g1, g2 = torch.Generator().manual_seed(3), torch.Generator().manual_seed(3)
    state = random.getstate()
    v, pix = batches.draw_source_view(5, 10, 12, view=4, ray_batch_size=20, generator=g1)
    assert random.getstate() == state                                                 # a given view draws nothing from `random`
    assert v == 4 and torch.equal(pix, 4 * 120 + torch.randint(0, 120, (20,), generator=g2))
    with pytest.raises(ValueError):
        batches.draw_source_view(5, 10, 12, view=5)


def test_test_time_optimizer_setup():
    """configure_optimizers for --is_optimize (model.py:957-981): Adam (0.9, 0.999) at 5e-6 over every parameter, the spatial encoder
    frozen, it and every BatchNorm2d in eval mode; the rest of the model trains."""
    pytest.importorskip("torchvision")
    from neo360_b200 import NeRF_TP
    from neo360_b200.encoder import GridEncoder
    torch.manual_seed(0)
    net = NeRF_TP(num_coarse_samples=8, num_fine_samples=4, num_src_views=5, encoder=GridEncoder()).train()
    opt = training.test_time_optimizer(net)
    assert isinstance(opt, torch.optim.Adam) and len(opt.param_groups) == 1
    group = opt.param_groups[0]
    assert group["lr"] == 5e-6 and group["betas"] == (0.9, 0.999) and group["weight_decay"] == 0
    assert [id(p) for p in group["params"]] == [id(p) for p in net.parameters()]
    se = net.encoder.spatial_encoder
    frozen = {id(p) for p in se.parameters()}
    assert frozen and not any(p.requires_grad for p in se.parameters())
    assert all(p.requires_grad for p in net.parameters() if id(p) not in frozen)
    assert not any(m.training for m in se.modules())
    bns = [m for m in net.modules() if isinstance(m, torch.nn.BatchNorm2d)]
    assert len(bns) > len([m for m in se.modules() if isinstance(m, torch.nn.BatchNorm2d)]) and not any(m.training for m in bns)
    assert net.training and net.encoder.depth_fc.training and net.encoder.floorplan_convnet_xz[0].training
    # eval_modules=False: frozen all the same, modes untouched (a loop that calls model.train() afterwards)
    net2 = NeRF_TP(num_coarse_samples=8, num_fine_samples=4, num_src_views=5, encoder=GridEncoder()).train()
    opt2 = training.test_time_optimizer(net2, lr=5e-4, eval_modules=False)
    assert opt2.param_groups[0]["lr"] == 5e-4
    assert not any(p.requires_grad for p in net2.encoder.spatial_encoder.parameters()) and all(m.training for m in net2.modules())


def test_test_time_optimizer_without_an_encoder():
    """Feature maps handed in the batch (no encoder): every parameter trains."""
    from neo360_b200 import NeRF_TP
    net = NeRF_TP(num_coarse_samples=8, num_fine_samples=4, num_src_views=1).train()
    opt = training.test_time_optimizer(net)
    assert all(p.requires_grad for p in net.parameters()) and sum(len(g["params"]) for g in opt.param_groups) == len(list(net.parameters()))
