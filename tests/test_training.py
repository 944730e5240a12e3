"""Training path (SURVEY.md 8(f2), 8(e) training row): the assembled differentiable NeRF_TP.forward against the oracle's gradients and
the flat-buffer gradient all-reduce (gloo, CPU).  The hand-written backward stages on their own are checked against float64 in
tests/test_gpu_train_stages.py."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from neo360_b200 import synth
from oracle import neo360_oracle as orc


def md(a, b):
    return float((a.detach().cpu().double() - b.detach().cpu().double()).abs().max())


@pytest.fixture(scope="module")
def cuda():
    assert torch.cuda.is_available()
    from neo360_b200 import build
    build.build()
    return torch.device("cuda:0")


def _tiny(cuda, nv=3):
    from neo360_b200 import NeRF_TP
    W, H, nc, nf = 32, 24, 8, 4
    sc = synth.make_scene((W, H), nv, (12, 16), 7)
    P = synth.make_mlp_params(7)
    net = NeRF_TP(num_coarse_samples=nc, num_fine_samples=nf, num_src_views=nv, precision="fp32")
    net.load_state_dict(P)
    net = net.to(cuda).train()
    pose = synth.target_pose(5, 100)
    ro, vd, rd, _ = orc.rays_from_pose(orc.ray_directions(H, W, 0.8 * W), pose[:3, :4])
    sel = torch.arange(100, 100 + 24)
    rays = {"rays_o": ro[sel].contiguous(), "rays_d": rd[sel].contiguous(), "viewdirs": vd[sel].contiguous()}
    return net, sc, P, rays, (W, H, nc, nf)


@pytest.mark.gpu
@pytest.mark.parametrize("projected", [True, False])
def test_training_forward_and_gradients_vs_oracle(cuda, projected):
    """NeRF_TP.forward in training mode: the train tuples (model.py:577-579) equal the oracle's, and the gradients of
    MSE + distortion loss w.r.t. EVERY MLP parameter, the tri-planes and the latent equal autograd through the oracle (CPU, fp32).
    Both formulations: `projected` (default: map columns of layers 0 / 3 applied to the feature maps, lookups of the projected maps through
    neo_index_maps / neo_index_maps_bwd) and the reference's row-by-row one.
    Stated: tuples 2e-4; every gradient tensor within 1e-2 of its gradient scale in max norm and 3e-3 in relative L2 (fp32 summation order)."""
    from neo360_b200 import training
    net, sc, P, rays, (W, H, nc, nf) = _tiny(cuda)
    net.train_projected = projected
    Pg = {k: v.clone().requires_grad_(True) for k, v in P.items()}
    maps = {k: sc[k].clone().requires_grad_(True) for k in ("planes_xz", "planes_xy", "planes_yz", "latent")}
    osc = orc.Scene(maps["planes_xz"], maps["planes_xy"], maps["planes_yz"], maps["latent"], sc["src_poses"],
                    float(sc["src_focal"][0]), float(sc["src_c"][0, 0]), float(sc["src_c"][0, 1]), W, H)
    target = torch.rand(rays["rays_o"].shape[0], 3, generator=torch.Generator().manual_seed(9))
    ref = orc.render(rays, osc, Pg, nc, nf, white_bkgd=False, out_depth=False)
    training.training_loss(ref, target).backward()

    dmaps = {k: sc[k].to(cuda).requires_grad_(True) for k in maps}
    batch = {k: v.to(cuda) for k, v in rays.items()}
    batch.update(dmaps)
    batch.update({k: sc[k].to(cuda) for k in ("src_poses", "src_focal", "src_c")})
    batch["src_imgs"] = torch.zeros(3, 3, H, W, device=cuda)
    got = net(batch, False, False, None, None, out_depth=False)
    for lvl in range(2):
        for a, b in zip(got[lvl], ref[lvl]):
            assert md(a, b) < 2e-4, (lvl, md(a, b))
    training.training_loss(got, target.to(cuda)).backward()
    # two measures per tensor: max |error| against the tensor's gradient scale (re-association noise of fp32 sums over ~1e5 point-views:
    # scatter-add atomics, GPU vs CPU GEMM order; bound 1e-2) and the relative L2 error of the whole tensor (bound 3e-3)
    rel2 = lambda a, b: float((a.detach().cpu().double() - b.detach().cpu().double()).norm() / max(float(b.detach().cpu().double().norm()), 1e-30))
    worst, worst2 = 0.0, 0.0
    for name, p in net.named_parameters():
        gref = Pg[name].grad
        scale = float(gref.abs().max())
        err, e2 = md(p.grad, gref), rel2(p.grad, gref)
        worst, worst2 = max(worst, err / max(scale, 1e-12)), max(worst2, e2)
        assert err < 1e-2 * scale + 1e-9 and e2 < 3e-3, (name, err, scale, e2)
    for k in maps:
        scale = float(maps[k].grad.abs().max())
        err, e2 = md(dmaps[k].grad, maps[k].grad), rel2(dmaps[k].grad, maps[k].grad)
        worst, worst2 = max(worst, err / max(scale, 1e-12)), max(worst2, e2)
        assert err < 1e-2 * scale + 1e-9 and e2 < 3e-3, (k, err, scale, e2)
    print(f"projected={projected}: worst max-abs gradient error / scale {worst:.2e}, worst relative L2 {worst2:.2e}")


@pytest.mark.gpu
def test_render_after_a_training_step_repacks_the_scene(cuda):
    """A training step leaves a cameras-only scene behind (projected formulation) and changes the weights: the next eval call on the same
    `set_scene` inputs must re-pack the scene for rendering and use the NEW weights (against the oracle, fp32 path, 2e-4)."""
    from neo360_b200 import training
    net, sc, P, rays, (W, H, nc, nf) = _tiny(cuda)
    dev_sc = [sc[k].to(cuda) for k in ("planes_xz", "planes_xy", "planes_yz", "latent", "src_poses", "src_focal", "src_c")]
    net.set_scene(*dev_sc, sc["img_wh"])
    batch = {k: v.to(cuda) for k, v in rays.items()}
    target = torch.rand(rays["rays_o"].shape[0], 3, generator=torch.Generator().manual_seed(3)).to(cuda)
    opt = torch.optim.SGD([p for m in net._mlps() for p in m.parameters()], lr=5e-2)
    loss = training.training_loss(net(batch, False, False, None, None, out_depth=False), target)
    loss.backward()
    opt.step()
    assert net._scene.mask == 0                                  # what the training step left
    net.eval()
    with torch.no_grad():
        got = net(batch, False, False, None, None, out_depth=True)[1]
    net.check()
    P2 = {k: v.detach().cpu() for k, v in net.state_dict().items()}
    osc = orc.Scene(sc["planes_xz"], sc["planes_xy"], sc["planes_yz"], sc["latent"], sc["src_poses"],
                    float(sc["src_focal"][0]), float(sc["src_c"][0, 0]), float(sc["src_c"][0, 1]), W, H)
    ref = orc.render(rays, osc, P2, nc, nf, False, True)[1]
    assert md(got[0], ref[0]) < 2e-4 and md(got[0], orc.render(rays, osc, P, nc, nf, False, True)[1][0]) > 1e-6


def _worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from neo360_b200.training import allreduce_flat
    ps = [torch.nn.Parameter(torch.zeros(3, 4)), torch.nn.Parameter(torch.zeros(5))]
    ps[0].grad = torch.full((3, 4), float(rank + 1))
    ps[1].grad = torch.arange(5.0) * (rank + 1)
    flat = allreduce_flat(ps, world, dist)
    q.put((rank, ps[0].grad.clone(), ps[1].grad.clone(), flat.numel()))
    dist.destroy_process_group()


def test_flat_gradient_allreduce_gloo():
    """allreduce_flat: one collective over the flat gradient slab, mean over ranks, written back into every .grad (world 2, gloo)."""
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(30)
    for rank, g0, g1, n in res:
        assert n == 17
        assert torch.allclose(g0, torch.full((3, 4), 1.5)) and torch.allclose(g1, torch.arange(5.0) * 1.5)


def test_distortion_loss_matches_quadratic_form():
    """The O(N) distortion loss equals the reference's in-tree O(N^2) lossfun_distortion (helper.py:111-118) on sorted midpoints with
    uniform intervals -- the functional eff_distloss implements (models/neo360/model.py:1246-1260)."""
    from neo360_b200.training import distortion_loss
    g = torch.Generator().manual_seed(0)
    B, N = 5, 17
    t = torch.sort(torch.rand(B, N + 1, generator=g), -1)[0]
    w = torch.rand(B, N, generator=g)
    m = 0.5 * (t[..., 1:] + t[..., :-1])
    dut = (m[..., :, None] - m[..., None, :]).abs()
    ref = ((w * (w[..., None, :] * dut).sum(-1)).sum(-1) + (w ** 2 * (t[..., 1:] - t[..., :-1])).sum(-1) / 3).mean()
    got = distortion_loss(w, m, t[..., 1:] - t[..., :-1])
    assert abs(float(got) - float(ref)) < 1e-6
