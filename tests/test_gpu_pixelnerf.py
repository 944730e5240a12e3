"""PixelNeRF on the CUDA path (neo360_b200.pixelnerf, csrc/pixelnerf.cu) against the golden vectors of the unmodified reference and
against float64 autograd through oracle/pixelnerf_oracle.py."""
import os

import numpy as np
import pytest
import torch

from neo360_b200 import synth
from oracle import pixelnerf_oracle as por

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "pixelnerf_reference_vectors.npz")
NEAR, FAR = 0.02, 3.0
DEV = torch.device("cuda:0")


def model(nv, nc, nf, seed):
    from neo360_b200 import PixelNeRF
    net = PixelNeRF(num_coarse_samples=nc, num_fine_samples=nf, num_src_views=nv)
    net.load_state_dict({**net.state_dict(), **synth.make_pixelnerf_params(seed)})
    return net.to(DEV)


def bypass(net, latent):
    """encoder(src_imgs) returns `latent` (the golden fixtures' synthetic encoder output)."""
    net.encoder.forward = lambda x: latent


def batch(rays, sc, focal=None, c=None):
    W, H = sc["img_wh"]
    nv = sc["src_poses"].shape[0]
    b = {k: v.to(DEV) for k, v in rays.items()}
    b.update(src_imgs=torch.zeros(nv, 3, H, W, device=DEV), src_poses=sc["src_poses"].to(DEV),
             src_focal=(sc["src_focal"] if focal is None else focal).to(DEV), src_c=(sc["src_c"] if c is None else c).to(DEV))
    return b


@pytest.mark.parametrize("tag", ("p1_b8", "p3_b8", "p3_b1024"))
def test_fp32_matches_golden(tag):
    z = np.load(GOLD)
    W, H, nv, B, nc, nf, seed = (int(x) for x in z[f"{tag}_cfg"])
    g = lambda k: torch.from_numpy(z[f"{tag}_{k}"])
    sc = synth.make_scene((W, H), nv, (8, 8), seed)
    net = model(nv, nc, nf, seed).eval()
    bypass(net, sc["latent"].to(DEV))
    b = batch({k: g(k) for k in ("rays_o", "rays_d", "viewdirs")}, sc, g("src_focal"), g("src_c"))
    with torch.no_grad():
        ev = net(b, False, True, NEAR, FAR)
        b["_uniforms"] = [g("u0").to(DEV), g("u1").to(DEV)]
        rr = net(b, True, False, NEAR, FAR)
    for lvl in range(2):
        for i, name in enumerate(("rgb", "acc", "depth")):
            for got, mode in ((ev, "eval"), (rr, "rand")):
                err = float((got[lvl][i].cpu() - g(f"{mode}{lvl}_{name}")).abs().max())
                assert err < 2e-4, (tag, mode, lvl, name, err)


def _oracle_case(nv, B, seed):
    W, H = 64, 48
    sc = synth.make_scene((W, H), nv, (8, 8), seed)
    from oracle import neo360_oracle as orc
    ro, vd, rd, _ = orc.rays_from_pose(orc.ray_directions(H, W, 0.8 * W), synth.target_pose(3, 100)[:3, :4])
    sel = torch.randperm(H * W, generator=torch.Generator().manual_seed(seed))[:B]
    rays = {"rays_o": ro[sel], "rays_d": rd[sel] * 0.7, "viewdirs": vd[sel]}
    return sc, rays, por.scene(sc["latent"], sc["src_poses"], sc["src_focal"], sc["src_c"], (W, H))


@pytest.mark.parametrize("nv", (1, 3, 5))
@pytest.mark.parametrize("randomized,white", ((False, False), (False, True), (True, False), (True, True)))
def test_fp32_matches_oracle(nv, randomized, white):
    """Every (randomized, white_bkgd) combination at NV 1, 3 and 5 against the float64 oracle, with injected uniforms: within 2e-4 plus
    twice the difference between the fp32 and float64 oracles on the same case."""
    B, nc, nf = 256, 32, 16
    sc, rays, osc = _oracle_case(nv, B, 11 + nv)
    g = torch.Generator().manual_seed(nv)
    rnd = {"u0": torch.rand(B, nc + 1, generator=g), "u1": torch.rand(B, nf, generator=g)} if randomized else None
    net = model(nv, nc, nf, 11).eval()
    bypass(net, sc["latent"].to(DEV))
    b = batch(rays, sc)
    if randomized:
        b["_uniforms"] = [rnd["u0"].to(DEV), rnd["u1"].to(DEV)]
    P = synth.make_pixelnerf_params(11)
    d64 = lambda x: None if x is None else {k: v.double() for k, v in x.items()}
    with torch.no_grad():
        got = net(b, randomized, white, NEAR, FAR)
        ref32 = por.render(rays, osc, P, nc, nf, NEAR, FAR, white, rand=rnd)
        ref = por.render(d64(rays), dict(osc, latent=osc["latent"].double(), src_poses=osc["src_poses"].double()), d64(P), nc, nf, NEAR,
                         FAR, white, rand=d64(rnd))
    for lvl in range(2):
        for i in range(3):
            # the fine level resamples from the coarse weights; where that is ill-conditioned (measured up to 2.4e-4 at NV = 1 between the
            # fp32 and float64 oracles) the bound widens by twice the case's own fp32-vs-float64 difference
            cond = float((ref32[lvl][i].double() - ref[lvl][i]).abs().max())
            err = float((got[lvl][i].cpu().double() - ref[lvl][i]).abs().max())
            assert err < 2e-4 + 2 * cond, (lvl, i, err, cond)


@pytest.mark.parametrize("nv", (1, 3, 5))
def test_tc_field_matches_fp16_model(nv):
    """precision="tc": sigma / rgb of every point of both levels against the float64 model of its fp16 numerics
    (oracle/pixelnerf_tc_model.py, bounds RGB_TOL / SIGMA_TOL and their means), at the fp32 path's own sample distances."""
    from oracle import pixelnerf_tc_model as ptm
    B, nc, nf = 512, 64, 64
    sc, rays, osc = _oracle_case(nv, B, 21 + nv)
    P = synth.make_pixelnerf_params(21)
    net = model(nv, nc, nf, 21).eval()
    bypass(net, sc["latent"].to(DEV))
    b = batch(rays, sc)
    g = torch.Generator().manual_seed(5)
    t0 = torch.sort(NEAR + (FAR - NEAR) * torch.rand(B, nc + 1, generator=g), -1).values
    t1 = torch.sort(NEAR + (FAR - NEAR) * torch.rand(B, nc + 1 + nf, generator=g), -1).values
    net.precision = "tc"
    for lvl, t in enumerate((t0, t1)):
        rgb, sigma = net.field(b, t.to(DEV), lvl)
        m_rgb, m_sigma = ptm.tc_field(P, ("coarse_mlp.", "fine_mlp.")[lvl], rays, t, osc)
        e = ptm.errors(rgb, sigma, m_rgb, m_sigma)
        print(f"pixelnerf tc nv={nv} level {lvl}: rgb max {e[0]:.2e} mean {e[1]:.2e}, sigma max {e[2]:.2e} mean {e[3]:.2e}")
        assert e[0] <= ptm.RGB_TOL and e[1] <= ptm.RGB_MEAN_TOL, e
        assert e[2] <= ptm.SIGMA_TOL and e[3] <= ptm.SIGMA_MEAN_TOL, e


def test_tc_frame_against_fp32():
    """A 640x480 frame (NV = 3, 64+64 samples) in "tc" against "fp32": PSNR of the fine rgb >= 66 dB (72.0 dB measured on an H100), and
    the weights re-packed when `precision` changes."""
    W, H, nv, nc, nf = 640, 480, 3, 64, 64
    sc = synth.make_scene((W, H), nv, (8, 8), 4)
    from oracle import neo360_oracle as orc
    ro, vd, rd, _ = orc.rays_from_pose(orc.ray_directions(H, W, 0.8 * W), synth.target_pose(5, 100)[:3, :4])
    net = model(nv, nc, nf, 4).eval()
    bypass(net, sc["latent"].to(DEV))
    b = batch({"rays_o": ro, "rays_d": rd, "viewdirs": vd}, sc)
    out = {}
    with torch.no_grad():
        for prec in ("fp32", "tc", "fp32"):
            net.precision = prec
            out.setdefault(prec, []).append(net(b, False, False, NEAR, FAR, chunk=4096)[1][0])
    assert torch.equal(out["fp32"][0], out["fp32"][1])
    mse = float(((out["tc"][0] - out["fp32"][0]) ** 2).mean())
    psnr = -10 * np.log10(max(mse, 1e-20))
    print(f"pixelnerf tc frame vs fp32: PSNR {psnr:.1f} dB, max {float((out['tc'][0] - out['fp32'][0]).abs().max()):.2e}")
    assert psnr >= 66.0


def test_frame_chunking_only_changes_through_q1():
    """A 640x480 frame rendered in one call with chunk=C equals C-ray calls one by one, bit for bit: the only coupling between rays is
    the reproduced quirk Q1."""
    W, H, nv, nc, nf = 640, 480, 3, 64, 64
    sc = synth.make_scene((W, H), nv, (8, 8), 4)
    from oracle import neo360_oracle as orc
    ro, vd, rd, _ = orc.rays_from_pose(orc.ray_directions(H, W, 0.8 * W), synth.target_pose(5, 100)[:3, :4])
    net = model(nv, nc, nf, 4).eval()
    bypass(net, sc["latent"].to(DEV))
    b = batch({"rays_o": ro, "rays_d": rd, "viewdirs": vd}, sc)
    C = 4096
    with torch.no_grad():
        whole = net(b, False, False, NEAR, FAR, chunk=C)
        parts = [net({**b, **{k: b[k][i:i + C] for k in ("rays_o", "rays_d", "viewdirs")}}, False, False, NEAR, FAR)
                 for i in range(0, W * H, C)]
        other = net(b, False, False, NEAR, FAR, chunk=1024)
    for lvl in range(2):
        for i in range(3):
            assert torch.equal(whole[lvl][i], torch.cat([p[lvl][i] for p in parts])), (lvl, i)
    assert not torch.equal(whole[1][0], other[1][0])            # Q1 does depend on the chunk size


def _train_case(nv=3, B=64, nc=16, nf=8, seed=6, W=64, H=48):
    sc = synth.make_scene((W, H), nv, (8, 8), seed)
    from oracle import neo360_oracle as orc
    ro, vd, rd, _ = orc.rays_from_pose(orc.ray_directions(H, W, 0.8 * W), synth.target_pose(2, 100)[:3, :4])
    g = torch.Generator().manual_seed(seed)
    sel = torch.randperm(H * W, generator=g)[:B]
    rays = {"rays_o": ro[sel], "rays_d": rd[sel], "viewdirs": vd[sel]}
    u = [torch.rand(B, nc + 1, generator=g), torch.rand(B, nf, generator=g)]
    target = torch.rand(B, 3, generator=g)
    return sc, rays, u, target


def _oracle_grads(net, rays, sc, latent, u, target, nc, nf, W, H, encoder=None, imgs=None):
    P = {k: v.detach().cpu().double().requires_grad_(True) for k, v in net.state_dict().items() if "mlp" in k}
    if encoder is None:
        lat = latent.detach().cpu().double().requires_grad_(True)
        lat_used = lat
    else:
        lat = None
        lat_used = encoder(imgs)
    osc = por.scene(lat_used, sc["src_poses"].double(), sc["src_focal"], sc["src_c"], (W, H))
    r64 = {k: v.double() for k, v in rays.items()}
    ret = por.render(r64, osc, P, nc, nf, NEAR, FAR, False, rand={"u0": u[0].double(), "u1": u[1].double()})
    loss = ((ret[0][0] - target.double()) ** 2).mean() + ((ret[1][0] - target.double()) ** 2).mean()
    loss.backward()
    return P, lat


def _close(a, b, what, rel=2e-3):
    err, scale = float((a.double().cpu() - b.double()).abs().max()), float(b.abs().max())
    assert err <= rel * scale + 1e-7, (what, err, scale)


def test_training_gradients_match_float64_oracle():
    """Gradients of every MLP parameter and of the latent: the CUDA training step against float64 autograd through the oracle, within
    5e-3 of each tensor's largest gradient.  The fine level resamples from fp32 weights here and float64 weights there, so its sample
    positions differ by fp32 rounding; that moves the fine MLP's gradients by up to 3e-3 of their scale (measured on an H100)."""
    torch.backends.cuda.matmul.allow_tf32 = False
    nv, B, nc, nf, W, H = 3, 64, 16, 8, 64, 48
    sc, rays, u, target = _train_case(nv, B, nc, nf, 6, W, H)
    net = model(nv, nc, nf, 6).train()
    latent = sc["latent"].to(DEV).requires_grad_(True)
    bypass(net, latent)
    b = batch(rays, sc)
    b["_uniforms"] = [x.to(DEV) for x in u]
    ret = net(b, True, False, NEAR, FAR)
    t = target.to(DEV)
    (((ret[0][0] - t) ** 2).mean() + ((ret[1][0] - t) ** 2).mean()).backward()
    P, lat = _oracle_grads(net, rays, sc, latent, u, target, nc, nf, W, H)
    named = dict(net.named_parameters())
    for k, p in P.items():
        _close(named[k].grad, p.grad, k, rel=5e-3)
    _close(latent.grad, lat.grad, "latent", rel=5e-3)


def test_training_gradients_real_encoder():
    """The same with the real ResNet-34 trunk (random weights, train-mode batch norm): its parameters' gradients too."""
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    nv, B, nc, nf, W, H = 2, 64, 16, 8, 64, 48
    sc, rays, u, target = _train_case(nv, B, nc, nf, 8, W, H)
    torch.manual_seed(8)
    net = model(nv, nc, nf, 8).train()
    enc64 = __import__("copy").deepcopy(net.encoder).cpu().double().train()
    imgs = torch.rand(nv, 3, H, W, generator=torch.Generator().manual_seed(1))
    b = batch(rays, sc)
    b["src_imgs"] = imgs.to(DEV)
    b["_uniforms"] = [x.to(DEV) for x in u]
    ret = net(b, True, False, NEAR, FAR)
    t = target.to(DEV)
    (((ret[0][0] - t) ** 2).mean() + ((ret[1][0] - t) ** 2).mean()).backward()
    P, _ = _oracle_grads(net, rays, sc, None, u, target, nc, nf, W, H, encoder=enc64, imgs=imgs.double())
    named = dict(net.named_parameters())
    for k, p in P.items():
        _close(named[k].grad, p.grad, k)
    for k, p in enc64.named_parameters():
        _close(named["encoder." + k].grad, p.grad, "encoder." + k, rel=5e-3)


def test_deterministic_training_steps_are_bit_identical():
    nv, B, nc, nf, W, H = 3, 256, 16, 8, 64, 48
    sc, rays, u, target = _train_case(nv, B, nc, nf, 9, W, H)
    imgs = torch.rand(nv, 3, H, W, generator=torch.Generator().manual_seed(2)).to(DEV)
    finals = []
    torch.use_deterministic_algorithms(True)
    try:
        for _ in range(2):
            torch.manual_seed(0)
            net = model(nv, nc, nf, 9).train()
            opt = torch.optim.Adam(net.parameters(), lr=5e-4)
            b = batch(rays, sc)
            b["src_imgs"] = imgs
            b["_uniforms"] = [x.to(DEV) for x in u]
            for _ in range(2):
                ret = net(b, True, False, NEAR, FAR)
                t = target.to(DEV)
                loss = ((ret[0][0] - t) ** 2).mean() + ((ret[1][0] - t) ** 2).mean()
                opt.zero_grad()
                loss.backward()
                opt.step()
            finals.append({k: v.detach().clone() for k, v in net.state_dict().items()})
    finally:
        torch.use_deterministic_algorithms(False)
    for k in finals[0]:
        assert torch.equal(finals[0][k], finals[1][k]), k


def test_state_dict_round_trip_and_optimizer_step_repacks():
    nv, nc, nf, W, H = 3, 16, 8, 64, 48
    sc = synth.make_scene((W, H), nv, (8, 8), 12)
    _, rays, _, target = _train_case(nv, 128, nc, nf, 12, W, H)
    imgs = torch.rand(nv, 3, H, W, generator=torch.Generator().manual_seed(3)).to(DEV)
    torch.manual_seed(1)
    a = model(nv, nc, nf, 12).eval()
    b_ = batch(rays, sc)
    b_["src_imgs"] = imgs
    with torch.no_grad():
        before = a(b_, False, False, NEAR, FAR)
    from neo360_b200 import PixelNeRF
    c = PixelNeRF(num_coarse_samples=nc, num_fine_samples=nf, num_src_views=nv).to(DEV).eval()
    sd = {k: v.cpu() for k, v in a.state_dict().items()}
    assert any(k.startswith("encoder.model.layer3.") for k in sd) and "coarse_mlp.pts_linears.0.weight" in sd
    with torch.no_grad():
        c(b_, False, False, NEAR, FAR)                          # packs c's own (different) weights first
    c.load_state_dict(sd)
    with torch.no_grad():
        after = c(b_, False, False, NEAR, FAR)
    for lvl in range(2):
        for i in range(3):
            assert torch.equal(before[lvl][i], after[lvl][i])
    c.train()
    opt = torch.optim.SGD(c.parameters(), lr=1.0)
    ret = c(b_, False, False, NEAR, FAR)
    (((ret[1][0] - target.to(DEV)) ** 2).mean()).backward()
    opt.step()
    c.eval()
    with torch.no_grad():
        stepped = c(b_, False, False, NEAR, FAR)
    ref = por.render({k: v for k, v in rays.items()},
                     por.scene(c.encoder(imgs).detach().cpu(), sc["src_poses"], sc["src_focal"], sc["src_c"], (W, H)),
                     {k: v.detach().cpu() for k, v in c.state_dict().items() if "mlp" in k}, nc, nf, NEAR, FAR, False)
    assert not torch.equal(stepped[1][0], after[1][0])
    assert float((stepped[1][0].cpu() - ref[1][0]).abs().max()) < 2e-4


def test_rejects_non_reference_options():
    from neo360_b200 import PixelNeRF
    for kw in ({"noise_std": 1.0}, {"lindisp": True}, {"num_levels": 3}):
        with pytest.raises(NotImplementedError):
            PixelNeRF(**kw)
    net = PixelNeRF().to(DEV).eval()
    net.precision = "bf16"
    with pytest.raises(ValueError):
        net({}, False, False, NEAR, FAR)
