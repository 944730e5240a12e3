"""GPU: NeO-360 at 1 and 5 source views (the reference's few-view settings) and its test-time optimisation.

At NV = 1 and 5, with the tolerances of the NV = 3 tests in tests/test_gpu_parity.py, tests/test_training.py and tests/test_gpu_mesh.py:
* fp32 end to end (eval, train and randomized tuples) against golden vectors of the UNMODIFIED reference (oracle/make_golden_views.py);
* tc end to end: PSNR >= 40 dB, L-inf 3e-2, and its randomized path with the reference's uniforms;
* a chunked frame against the oracle's chunk loop (quirk Q1);
* training gradients of both formulations and of the tc trunk against autograd through the oracle;
* the fp32 density grid; `field_eval` fp32 at NV = 6, 7 and 8 (4 points per CTA above 6 views).
Test-time optimisation (`training.test_time_optimizer`, `batches.source_view_batch`) with the encoder inside the step: the frozen parts
stay bit-identical, the ResNet runs once, each update is an unclipped constant-lr Adam step, and the loss on the chosen view falls."""
import os

import numpy as np
import pytest
import torch

from neo360_b200 import synth
from oracle import field_train_model as ftm
from oracle import neo360_oracle as orc

pytestmark = pytest.mark.gpu
T = lambda a: torch.from_numpy(np.asarray(a))
EV = ("comp_rgb", "fg_rgb", "bg_rgb", "fg_acc", "bg_lambda", "depth")
TR = ("comp_rgb", "fg_w", "bg_w", "fg_sdist", "bg_sdist", "bg_acc")
TAGS = ["nv1_tiny", "nv5_tiny", "nv5_small"]
MAPS = ("planes_xz", "planes_xy", "planes_yz", "latent")
SRC = ("src_poses", "src_focal", "src_c")


@pytest.fixture(scope="module")
def cuda():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from neo360_b200 import build
    build.build()
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def vgolden():
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "neo360_views_vectors.npz"))


def md(a, b):
    return float((a.detach().cpu().double() - b.detach().cpu().double()).abs().max())


def oracle_scene(sc, W, H, maps=None):
    m = maps or sc
    return orc.Scene(m["planes_xz"], m["planes_xy"], m["planes_yz"], m["latent"], sc["src_poses"], float(sc["src_focal"][0]),
                     float(sc["src_c"][0, 0]), float(sc["src_c"][0, 1]), W, H)


def make_net(cuda, nv, img_wh, plane_hw, nc, nf, seed, precisions=("fp32",), precision="fp32"):
    from neo360_b200 import NeRF_TP
    sc = synth.make_scene(img_wh, nv, plane_hw, seed)
    P = synth.make_mlp_params(seed)
    net = NeRF_TP(num_coarse_samples=nc, num_fine_samples=nf, num_src_views=nv, precision=precision).eval()
    net.load_state_dict(P)
    net = net.to(cuda)
    net.set_scene(*[sc[k].to(cuda) for k in MAPS + SRC], sc["img_wh"], precisions=list(precisions))
    return net, oracle_scene(sc, *img_wh), P


def golden_case(cuda, g, tag, **kw):
    W, H, hp, wp, B, nc, nf, seed, start = [int(x) for x in g[f"{tag}_cfg"]]
    net, osc, P = make_net(cuda, int(g[f"{tag}_nv"]), (W, H), (hp, wp), nc, nf, seed, **kw)
    rays = {k: T(g[f"{tag}_{k}"]).to(cuda) for k in ("rays_o", "rays_d", "viewdirs")}
    rays_r = dict(rays)
    rays_r["_uniforms"] = [T(g[f"{tag}_u_{k}"]).to(cuda) for k in ("fg0", "bg0", "fg1", "bg1")]
    return net, rays, rays_r


@pytest.mark.parametrize("tag", TAGS)
def test_end_to_end_fp32_vs_reference_vectors(cuda, vgolden, tag):
    """Tolerance of the NV = 3 test: 2e-4 on every output, up to 1 % of entries beyond it (quirk Q17) bounded by 5e-3."""
    g = vgolden
    net, rays, rays_r = golden_case(cuda, g, tag)
    with torch.no_grad():
        ev = net(rays, False, False, 0.2, 3.0, out_depth=True, debug=True)
        dbg = net.last_debug
        tr = net(rays, False, True, 0.2, 3.0, out_depth=False)
        rr = net(rays_r, True, False, 0.2, 3.0, out_depth=True)
    net.check()

    def close(v, ref, name):
        diff = (v.cpu().double() - T(ref).double()).abs()
        assert float(diff.max()) < 5e-3, (name, float(diff.max()))
        assert float((diff > 2e-4).double().mean()) <= 0.01, (name, float(diff.max()))

    for lvl in range(2):
        for names, got, kind in ((EV, ev, "eval"), (TR, tr, "train"), (EV, rr, "rand")):
            for n_, v in zip(names, got[lvl]):
                close(v, g[f"{tag}_{kind}{lvl}_{n_}"], (kind, lvl, n_))
    for k, dk in (("fg_t", "fg_t"), ("fg_sigma", "fg_sigma"), ("fg_rgb", "fg_rgb_s")):
        close(dbg[dk][0].reshape(g[f"{tag}_aux0_{k}"].shape), g[f"{tag}_aux0_{k}"], ("aux", k))


@pytest.mark.parametrize("tag", TAGS)
def test_end_to_end_tc_vs_reference_vectors(cuda, vgolden, tag):
    """Bounds of the NV = 3 test: L-inf 3e-2 on every eval output and PSNR >= 40 dB on comp_rgb; randomized with the reference's
    uniforms and the train tuple within 3e-2, coarse sdist exact to 1e-6."""
    g = vgolden
    net, rays, rays_r = golden_case(cuda, g, tag, precisions=("tc",), precision="tc")
    with torch.no_grad():
        ev = net(rays, False, False, 0.2, 3.0, out_depth=True)
        rr = net(rays_r, True, False, 0.2, 3.0, out_depth=True)
        tr = net(rays, False, True, 0.2, 3.0, out_depth=False)
    net.check()
    for lvl in range(2):
        for n_, v in zip(EV, ev[lvl]):
            assert md(v, T(g[f"{tag}_eval{lvl}_{n_}"])) < 3e-2, (lvl, n_)
        assert md(rr[lvl][0], T(g[f"{tag}_rand{lvl}_comp_rgb"])) < 3e-2, lvl
    ps = orc.psnr(ev[1][0].cpu(), T(g[f"{tag}_eval1_comp_rgb"]))
    print(f"tc [{tag}]: PSNR {ps:.1f} dB")
    assert ps > 40
    assert md(tr[0][3], T(g[f"{tag}_train0_fg_sdist"])) < 1e-6
    assert md(tr[0][1], T(g[f"{tag}_train0_fg_w"])) < 3e-2 and md(tr[1][0], T(g[f"{tag}_train1_comp_rgb"])) < 3e-2


def frame_rays(W, H, view=11):
    pose = synth.target_pose(view, 100)
    ro, vd, rd, _ = orc.rays_from_pose(orc.ray_directions(H, W, 0.8 * W), pose[:3, :4])
    return {"rays_o": ro, "rays_d": rd, "viewdirs": vd}


@pytest.mark.parametrize("nv", [1, 5])
def test_chunked_frame_matches_oracle_chunk_loop(cuda, nv):
    """A 48x36 frame in one call with chunk = 512 against the oracle's loop over 512-ray chunks (last chunk ragged), fp32 and tc."""
    W, H, nc, nf = 48, 36, 24, 12
    net, osc, P = make_net(cuda, nv, (W, H), (24, 32), nc, nf, 2, precisions=("fp32", "tc"))
    rays = frame_rays(W, H)
    cr = {k: v.to(cuda) for k, v in rays.items()}
    with torch.no_grad():
        ref = orc.render_chunked(rays, osc, P, nc, nf, chunk=512)
        got = net.render_rays_test(cr, chunk=512)
        net.precision = "tc"
        tc = net.render_rays_test(cr, chunk=512, img_wh=(W, H))
    net.check()
    for k in ("rgb", "fg_rgb", "bg_rgb", "depth"):
        diff = (got[k].cpu() - ref["comp_rgb" if k == "rgb" else k]).abs()
        assert float(diff.max()) < 5e-3 and float((diff > 2e-4).float().mean()) < 0.01, (k, float(diff.max()))
    assert orc.psnr(got["rgb"].cpu(), ref["comp_rgb"]) > 60
    assert md(tc["rgb"], ref["comp_rgb"]) < 3e-2 and orc.psnr(tc["rgb"].cpu(), ref["comp_rgb"]) > 40


@pytest.mark.parametrize("nv", [1, 5])
@pytest.mark.parametrize("form", ["projected", "reference", "tc"])
def test_training_gradients_vs_oracle(cuda, nv, form):
    """The training-mode forward and the gradients of MSE + distortion loss with respect to every MLP parameter and the feature maps,
    against autograd through the oracle.  fp32 formulations: tuples 2e-4 (as at NV = 3, tests/test_training.py); every gradient tensor
    within 5e-2 of its gradient scale in max norm and 2e-2 in relative L2.  That is looser than the NV = 3 test's 1e-2 / 3e-3: measured
    on an H100, the worst tensors reach 4.4e-3 (NV = 1) and 1.1e-2 (NV = 5) in relative L2, and 3.3e-2 of the scale in max norm
    (bg_coarse_mlp.pts_linears.2.weight, NV = 5), and both formulations give the same errors to 8 digits.  So the difference comes from what they share -- sample points, camera
    transforms and positional encodings, whose top frequency (2^9) magnifies last-bit differences -- not from the lookups or layers.
    tc trunk: the coarse level's tuple within 3e-2; the coarse MLPs' gradients within the whole-step
    bound of tests/test_gpu_field_train.py (oracle/field_train_model.STEP_BOUND).  The fine level's samples follow the bf16 coarse
    weights, so its gradients are compared with the fp32 path's there, on a 4096-ray step."""
    from neo360_b200 import NeRF_TP, training
    W, H, nc, nf = 32, 24, 8, 4
    sc = synth.make_scene((W, H), nv, (12, 16), 7)
    P = synth.make_mlp_params(7)
    net = NeRF_TP(num_coarse_samples=nc, num_fine_samples=nf, num_src_views=nv, precision="fp32",
                  train_precision="tc" if form == "tc" else "fp32")
    net.load_state_dict(P)
    net = net.to(cuda).train()
    net.train_projected = form != "reference"
    rays = {k: v[100:124].contiguous() for k, v in frame_rays(W, H, 5).items()}
    Pg = {k: v.clone().requires_grad_(True) for k, v in P.items()}
    maps = {k: sc[k].clone().requires_grad_(True) for k in MAPS}
    target = torch.rand(24, 3, generator=torch.Generator().manual_seed(9))
    ref = orc.render(rays, oracle_scene(sc, W, H, maps), Pg, nc, nf, white_bkgd=False, out_depth=False)
    training.training_loss(ref, target).backward()
    dmaps = {k: sc[k].to(cuda).requires_grad_(True) for k in MAPS}
    batch = {k: v.to(cuda) for k, v in rays.items()}
    batch.update(dmaps)
    batch.update({k: sc[k].to(cuda) for k in SRC})
    batch["src_imgs"] = torch.zeros(nv, 3, H, W, device=cuda)
    got = net(batch, False, False, None, None, out_depth=False)
    for lvl in range(2):
        for j, (a, b) in enumerate(zip(got[lvl], ref[lvl])):
            if form != "tc":
                assert md(a, b) < 2e-4, (lvl, j, md(a, b))
            elif lvl == 0:
                assert md(a, b) < 3e-2, (lvl, j, md(a, b))
    training.training_loss(got, target.to(cuda)).backward()
    pairs = [(n, p.grad, Pg[n].grad) for n, p in net.named_parameters()] + [(k, dmaps[k].grad, maps[k].grad) for k in MAPS]
    if form == "tc":
        pairs = [t for t in pairs if t[0].startswith(("fg_coarse_mlp.", "bg_coarse_mlp."))]
    rel = {name: ftm.rel_err(a.cpu(), b) for name, a, b in pairs}
    print(f"nv={nv} {form}: relative L2 gradient errors, largest first:", sorted(rel.items(), key=lambda kv: -kv[1])[:4])
    for name, a, b in pairs:
        if form == "tc":
            assert rel[name] < ftm.STEP_BOUND, (name, rel[name])
        else:
            scale = float(b.abs().max())
            assert md(a, b) < 5e-2 * scale + 1e-9 and rel[name] < 2e-2, (name, md(a, b), scale, rel[name])


@pytest.mark.parametrize("nv", [1, 5])
def test_density_grid_fp32_vs_oracle(cuda, nv):
    """The fp32 density grid (neo_field_eval per lattice row) within 2e-4 of the oracle's NeRFPPMLP, 0 outside the unit sphere."""
    from neo360_b200 import mesh
    from oracle import mesh_model as mm
    net, osc, P = make_net(cuda, nv, (64, 48), (24, 32), 8, 4, 0)
    box = ((-1.2, -1.1, -1.0), (1.0, 1.2, 1.1))
    shape = (13, 12, 14)
    sig = net.density_grid(shape, box, level=1, precision="fp32", slab_rays=100).cpu().reshape(-1)
    g = mesh.make_grid(shape, box)
    ax = [mm.lattice(list(g.origin), list(g.step), n, a, True) for a, n in enumerate((g.nx, g.ny, g.nz))]
    Z, Y, X = np.meshgrid(ax[2], ax[1], ax[0], indexing="ij")
    pts = torch.from_numpy(np.stack([X, Y, Z], -1).reshape(-1, 3))
    cam = orc.world2camera(pts, osc.src_poses)
    with torch.no_grad():
        _, raw = orc.mlp_forward(P, "fg_fine_mlp.", orc.pos_enc(cam, 0, 10), torch.zeros(nv * pts.shape[0], 27),
                                 orc.triplane_lookup(cam, osc).reshape(-1, 128), orc.local_lookup(cam, osc).reshape(-1, 512), nv)
    ref = torch.nn.functional.softplus(raw[:, 0] - 1.0)
    ref[(pts * pts).sum(-1) > 1] = 0
    assert float((sig - ref).abs().max()) < 2e-4 and float(ref.abs().max()) > 0.1


@pytest.mark.parametrize("nv", [6, 7, 8])
def test_field_eval_fp32_many_views(cuda, nv):
    """`field_eval` fp32 above 5 views (8 points per CTA at 6, 4 at 7 and 8) against the oracle on identical t-values, every branch, with
    a point count that leaves a partial tile.  Bound 1e-4, twice the NV = 3 test's: the worst measured on an H100 is 5.3e-5 in sigma
    (NV = 7), where the view mean sums seven rows."""
    nc = 16
    net, osc, P = make_net(cuda, nv, (64, 48), (24, 32), nc, 8, 0)
    rays = {k: v[1000:1000 + 41].contiguous() for k, v in frame_rays(64, 48, 3).items()}
    with torch.no_grad():
        _, aux = orc.render(rays, osc, P, nc, 8, False, True, return_aux=True)
    cr = {k: v.to(cuda) for k, v in rays.items()}
    for lvl in range(2):
        for b, (tk, rk, sk) in enumerate((("fg_t", "fg_rgb", "fg_sigma"), ("bg_s", "bg_rgb", "bg_sigma"))):
            rgb, sig = net.field_eval(cr, aux[lvl]["far"].to(cuda), aux[lvl][tk].to(cuda), 2 * lvl + b, precision="fp32")
            net.check()
            assert md(sig, aux[lvl][sk]) < 1e-4 and md(rgb, aux[lvl][rk]) < 1e-4, (nv, lvl, b, md(sig, aux[lvl][sk]), md(rgb, aux[lvl][rk]))


# ---------------- test-time optimisation ----------------

def tto_setup(cuda, nv, W=160, H=120, lr=None, constant=False):
    """A model with the encoder, as --is_optimize loads it, on a synthetic scene: NV source images (their own poses are the targets)."""
    from neo360_b200 import NeRF_TP, batches, training
    from neo360_b200.encoder import GridEncoder
    torch.manual_seed(0)
    net = NeRF_TP(num_coarse_samples=32, num_fine_samples=16, num_src_views=nv, precision="fp32", encoder=GridEncoder())
    sd = net.state_dict()
    sd.update(synth.make_mlp_params(0))
    net.load_state_dict(sd)
    net = net.to(cuda).train()
    sc = synth.make_scene((W, H), nv, (4, 4), 0)
    g = torch.Generator().manual_seed(5)
    imgs = torch.rand(nv, 3, H // 8, W // 8, generator=g)
    imgs = torch.nn.functional.interpolate(imgs, size=(H, W), mode="bilinear", align_corners=False).clamp(0, 1).to(cuda)   # smooth images
    if constant:
        imgs = torch.full_like(imgs, 0.8)
    views = batches.TargetViews(sc["src_poses"].to(cuda), imgs.permute(0, 2, 3, 1), float(sc["src_focal"][0]))
    src = {k: sc[k].to(cuda) for k in SRC}
    src["src_imgs"] = imgs * 2 - 1                                  # normalised as the dataset hands them over
    opt = training.test_time_optimizer(net) if lr is None else training.test_time_optimizer(net, lr=lr)
    return net, opt, views, src


def test_source_view_batch(cuda):
    """The sample's keys are train_batch's, its rays and colours are those pixels of the drawn source view; a second focal raises."""
    import random
    from neo360_b200 import batches, ops
    net, opt, views, src = tto_setup(cuda, 5)
    random.seed(3)
    torch.manual_seed(3)
    b = batches.source_view_batch(views, src)
    random.seed(3)
    torch.manual_seed(3)
    v, pix = batches.draw_source_view(5, views.H, views.W)
    o, vd, rd, rad, tgt = ops.sample_rays(pix.to(cuda), views.H, views.W, views.focal, views.poses, views.images)
    assert b["rays_o"].shape == (500, 3) and torch.equal(b["rays_o"], o) and torch.equal(b["target"], tgt)
    assert torch.equal(tgt, views.images[v].reshape(-1, 3)[(pix - v * views.H * views.W).to(cuda)])
    p = batches.source_view_batch(views, src, view=2, finetune_lpips=True)
    assert p["rays_o"].shape == (900, 3)
    bad = dict(src)
    bad["src_focal"] = src["src_focal"].clone()
    bad["src_focal"][1] += 1
    with pytest.raises(ValueError, match="focal"):
        batches.source_view_batch(views, bad)


@pytest.mark.parametrize("nv", [1, 5])
@pytest.mark.parametrize("train_precision", ["fp32", "tc"])
def test_test_time_steps(cuda, nv, train_precision):
    """K = 3 test-time steps with the encoder inside: the spatial encoder's parameters and every BatchNorm running statistic are
    bit-identical afterwards, the ResNet ran once, and every parameter update equals a plain Adam step at the constant lr computed
    (float64) from the same gradients -- no schedule, no clip, although the gradient norm is far above the reference's 0.05 clip."""
    from neo360_b200 import batches, training
    net, opt, views, src = tto_setup(cuda, nv)
    net.train_precision = train_precision
    net.encoder.train_precision = train_precision
    se = net.encoder.spatial_encoder
    frozen = {k: v.clone() for k, v in se.state_dict().items()}
    stats = {n: b.clone() for n, b in net.named_buffers() if "running_" in n or "num_batches" in n}
    calls = []
    hook = se.model.conv1.register_forward_hook(lambda *a: calls.append(1))
    lr, (b1, b2), eps = opt.param_groups[0]["lr"], opt.param_groups[0]["betas"], opt.param_groups[0]["eps"]
    params = [p for p in net.parameters() if p.requires_grad]
    m = [torch.zeros_like(p, dtype=torch.float64) for p in params]
    v = [torch.zeros_like(p, dtype=torch.float64) for p in params]
    g = torch.Generator().manual_seed(11)
    for step in range(1, 4):
        batch = batches.source_view_batch(views, src, generator=g)
        before = [p.detach().clone() for p in params]
        ret = net(batch, True, False, None, None, out_depth=False)
        loss = training.training_loss(ret, batch["target"])
        opt.zero_grad(set_to_none=True)
        loss.backward()
        grads = [p.grad.detach().double() for p in params]
        norm = float(torch.sqrt(sum((x ** 2).sum() for x in grads)))
        assert norm > 10 * 0.05, norm                                   # measured 0.74 - 0.80 at NV = 1
        opt.step()
        for i, (p, p0, gi) in enumerate(zip(params, before, grads)):
            m[i] = b1 * m[i] + (1 - b1) * gi
            v[i] = b2 * v[i] + (1 - b2) * gi * gi
            exp = p0.double() - (lr / (1 - b1 ** step)) * m[i] / (v[i].sqrt() / (1 - b2 ** step) ** 0.5 + eps)
            err = float((p.detach().double() - exp).abs().max())
            assert err <= 1e-3 * lr + 4 * float(torch.finfo(torch.float32).eps * p0.abs().max()), (step, i, err)
    hook.remove()
    torch.cuda.synchronize()
    assert len(calls) == 1, len(calls)
    assert all(torch.equal(se.state_dict()[k], t) for k, t in frozen.items())
    assert all(torch.equal(b, stats[n]) for n, b in net.named_buffers() if n in stats)
    assert se.latent.shape[0] == nv
    assert all(p.grad is None for p in se.parameters())


def test_test_time_optimisation_lowers_the_loss(cuda):
    """50 test-time steps (`training.test_time_step`) on 5 source views of one colour: the MSE of a fixed set of the chosen view's
    pixels, rendered deterministically, falls by more than 10 %.  lr 5e-4, the reference's rate when it does not resume from a
    checkpoint.  The weights are untrained, so the images are uniform: on random images 50 steps of an untrained model do not lower
    the loss reliably."""
    import random
    from neo360_b200 import batches, training
    net, opt, views, src = tto_setup(cuda, 5, lr=5e-4, constant=True)
    random.seed(0)
    torch.manual_seed(0)
    view = random.sample(range(5), 1)[0]
    probe = batches.source_view_batch(views, src, view=view, ray_batch_size=2048, generator=torch.Generator().manual_seed(1))

    def mse():
        with torch.no_grad():
            out = net(probe, False, False, None, None, out_depth=True)[1][0]
        return float(((out - probe["target"]) ** 2).mean())

    g = torch.Generator().manual_seed(2)
    start = mse()
    for _ in range(50):
        training.test_time_step(net, opt, batches.source_view_batch(views, src, view=view, generator=g))
    end = mse()
    print(f"test-time optimisation, 50 steps: view-{view} MSE {start:.5f} -> {end:.5f}")
    assert end < 0.9 * start, (start, end)
