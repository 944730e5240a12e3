"""TEST INFRASTRUCTURE ONLY -- golden vectors for the PixelNeRF renderer from the UNMODIFIED reference `PixelNeRF`
(models/vanilla_nerf/model_pixel.py:133-258), and the pin of oracle/pixelnerf_oracle.py against it, stage by stage.

Run where the reference tree exists:   python oracle/make_golden_pixelnerf.py
Writes tests/golden/pixelnerf_reference_vectors.npz (ray inputs, injected uniforms, stage taps and both levels' outputs; the latent and
the MLP weights are regenerated from seeds by `neo360_b200.synth`).

The encoder is bypassed as for NeO-360: `encoder.forward` installs a synthetic smoothed latent.  One extra case runs the reference's
real ResNet-34 trunk on random weights and checks that `neo360_b200.encoder.SpatialEncoder` loads its state dict and computes the same
latent and latent_scaling, so the package reuses that class for PixelNeRF."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_shim  # noqa: E402
from oracle import pixelnerf_oracle as por  # noqa: E402
from oracle.make_golden import RandQueue, maxdiff  # noqa: E402
from neo360_b200 import synth  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
# tag: (W, H, NV, B, n_coarse, n_fine, seed).  B = 8 and B = 1024 are the two caller chunk sizes of quirk Q1.
CASES = {"p1_b8": (64, 48, 1, 8, 16, 8, 0), "p3_b8": (64, 48, 3, 8, 16, 8, 1), "p3_b1024": (64, 48, 3, 1024, 64, 64, 2)}
NEAR, FAR = 0.02, 3.0          # datasets/nerds360_ae.py:274-275


def make_reference(ns, nc, nf, nv, seed):
    import torchvision
    orig = torchvision.models.resnet34

    def resnet34_nodl(*a, **k):           # pretrained=True would download ImageNet weights
        k.pop("pretrained", None)
        return orig(weights=None, **k)

    torchvision.models.resnet34 = resnet34_nodl
    try:
        torch.manual_seed(seed)
        net = ns.pix_model.PixelNeRF(num_coarse_samples=nc, num_fine_samples=nf, num_src_views=nv)
    finally:
        torchvision.models.resnet34 = orig
    return net.eval()


def bypass_encoder(net, latent):
    se = net.encoder

    def fwd(x):
        se.latent = latent
        ls = torch.tensor([latent.shape[-1], latent.shape[-2]], dtype=torch.float32)
        se.latent_scaling = ls / (ls - 1) * 2.0             # encoder.py:182-184
        return latent

    se.forward = fwd


def rays_for(ns, W, H, B, seed):
    pose = synth.target_pose(7, 100)
    dirs = ns.ray_utils.get_ray_directions(H, W, 0.8 * W)
    ro, vd, rd = ns.ray_utils.get_rays(dirs, pose[:3, :4], output_view_dirs=True)
    g = torch.Generator().manual_seed(70 + seed)
    sel = torch.randperm(H * W, generator=g)[:B]
    scale = 0.5 + torch.rand(B, 1, generator=g)            # un-normalised rays_d: PixelNeRF marches along rays_d
    return {"rays_o": ro[sel].contiguous(), "rays_d": (rd[sel] * scale).contiguous(), "viewdirs": vd[sel].contiguous()}, g


def batch(rays, sc):
    W, H = sc["img_wh"]
    nv = sc["src_poses"].shape[0]
    out = dict(rays)
    out.update(src_imgs=torch.zeros(nv, 3, H, W), src_poses=sc["src_poses"], src_focal=sc["src_focal"], src_c=sc["src_c"])
    return out


def stage_taps(ns, net, rays, sc, N_dummy=5):
    """Reference helpers of model_pixel.py:207-232 on the coarse samples of `rays` against the oracle's `stages`."""
    util, helper = ns.pix_util, ns.van_helper
    nv = sc["src_poses"].shape[0]
    net.encoder(None)                                      # installs the latent (bypassed encoder)
    t, samples = helper.sample_along_rays(rays["rays_o"], rays["rays_d"], N_dummy, NEAR, FAR, False, False)
    B, N, _ = samples.shape
    s = samples.reshape(-1, 3).unsqueeze(0)
    cam = util.world2camera(s, sc["src_poses"], nv)
    focal = sc["src_focal"][0].unsqueeze(-1).repeat((1, 2))
    uv = util.projection(cam, focal, sc["src_c"][0].unsqueeze(0), nv)
    lat = net.encoder.index(uv, None, torch.Tensor([sc["img_wh"][0], sc["img_wh"][1]])).transpose(1, 2).reshape(-1, 512)
    vdc = util.world2camera_viewdirs(rays["viewdirs"].unsqueeze(0), sc["src_poses"], nv)
    denc = helper.pos_enc(vdc, 0, 4)
    tile = torch.tile(denc[:, None, :], (1, N, 1)).reshape(-1, denc.shape[-1])
    osc = por.scene(sc["latent"], sc["src_poses"], sc["src_focal"], sc["src_c"], sc["img_wh"])
    st = por.stages(samples, rays["viewdirs"], osc, N)
    worst = max(maxdiff(st["p_cam"], cam), maxdiff(st["uv"], uv), maxdiff(st["latent"], lat),
                maxdiff(st["enc"], helper.pos_enc(cam, 0, 10)), maxdiff(st["dir_tile"], tile))
    assert worst < 1e-4, worst
    return {"cam": cam, "uv": uv, "latent": lat, "dir_tile": tile}, worst


def real_encoder(ns, out):
    """The reference's ResNet-34 trunk (random weights) against neo360_b200.encoder.SpatialEncoder with the same state dict."""
    from neo360_b200.encoder import SpatialEncoder
    W, H, nv = 64, 48, 2
    net = make_reference(ns, 8, 4, nv, 5)
    ours = SpatialEncoder().eval()
    ref_keys = set(net.encoder.state_dict().keys())
    assert ref_keys == set(ours.state_dict().keys()), sorted(ref_keys ^ set(ours.state_dict().keys()))[:10]
    ours.load_state_dict(net.encoder.state_dict())
    imgs = torch.rand(nv, 3, H, W, generator=torch.Generator().manual_seed(9))
    with torch.no_grad():
        lr, lo = net.encoder(imgs), ours(imgs)
    d = maxdiff(lr, lo)
    assert d < 1e-5 and torch.equal(net.encoder.latent_scaling, ours.latent_scaling.cpu()), (d, net.encoder.latent_scaling)
    # end to end with the real trunk: reference PixelNeRF.forward == oracle on the package encoder's latent
    sc = synth.make_scene((W, H), nv, (8, 8), 5)
    rays, _ = rays_for(ns, W, H, 64, 5)
    P = synth.make_pixelnerf_params(5)
    net.load_state_dict({**net.state_dict(), **P})
    b = batch(rays, sc)
    b["src_imgs"] = imgs
    with torch.no_grad():
        ref = net(b, False, False, NEAR, FAR)
        got = por.render(rays, por.scene(lo, sc["src_poses"], sc["src_focal"], sc["src_c"], (W, H)), P, 8, 4, NEAR, FAR, False)
    worst = max(maxdiff(a, c) for lvl in range(2) for a, c in zip(got[lvl], ref[lvl]))
    assert worst < 2e-4, worst
    print(f"pixelnerf[real encoder]: latent max|diff| = {d:.3e}, oracle vs reference max|diff| = {worst:.3e}")
    out["enc_latent_maxdiff"] = np.array([d, worst])


def main():
    ns = ref_shim.load()
    import importlib
    ns.pix_model = importlib.import_module("models.vanilla_nerf.model_pixel")
    ns.pix_util = importlib.import_module("models.vanilla_nerf.util")
    out = {}
    for tag, (W, H, nv, B, nc, nf, seed) in CASES.items():
        sc = synth.make_scene((W, H), nv, (8, 8), seed)
        sc["src_focal"] = sc["src_focal"] * torch.linspace(1.0, 1.3, nv)     # only src_focal[0] / src_c[0] may be used
        sc["src_c"] = sc["src_c"] + torch.arange(nv, dtype=torch.float32)[:, None] * 3.0
        P = synth.make_pixelnerf_params(seed)
        net = make_reference(ns, nc, nf, nv, seed)
        net.load_state_dict({**net.state_dict(), **P}, strict=True)
        bypass_encoder(net, sc["latent"])
        rays, g = rays_for(ns, W, H, B, seed)
        b = batch(rays, sc)
        taps, tw = stage_taps(ns, net, rays, sc)
        osc = por.scene(sc["latent"], sc["src_poses"], sc["src_focal"], sc["src_c"], (W, H))
        with torch.no_grad():
            ev = net(b, False, True, NEAR, FAR)
            rnd = {"u0": torch.rand(B, nc + 1, generator=g), "u1": torch.rand(B, nf, generator=g)}
            with RandQueue([rnd["u0"], rnd["u1"]]):
                rr = net(b, True, False, NEAR, FAR)
            o_ev = por.render(rays, osc, P, nc, nf, NEAR, FAR, True)
            o_rr = por.render(rays, osc, P, nc, nf, NEAR, FAR, False, rand=rnd)
        worst = max(maxdiff(a, c) for got, ref in ((o_ev, ev), (o_rr, rr)) for lvl in range(2) for a, c in zip(got[lvl], ref[lvl]))
        assert worst < 2e-4, worst
        print(f"pixelnerf[{tag}]: stages max|diff| = {tw:.3e}, oracle vs reference max|diff| = {worst:.3e}")
        out.update({f"{tag}_cfg": np.array([W, H, nv, B, nc, nf, seed]), f"{tag}_rays_o": rays["rays_o"], f"{tag}_rays_d": rays["rays_d"],
                    f"{tag}_viewdirs": rays["viewdirs"], f"{tag}_src_focal": sc["src_focal"], f"{tag}_src_c": sc["src_c"],
                    f"{tag}_u0": rnd["u0"], f"{tag}_u1": rnd["u1"]})
        if B <= 8:                                         # stage taps of the small chunks only (the file stays small)
            for k, v in taps.items():
                out[f"{tag}_stage_{k}"] = v
        for lvl in range(2):
            for n_, a, c in zip(("rgb", "acc", "depth"), ev[lvl], rr[lvl]):
                out[f"{tag}_eval{lvl}_{n_}"] = a
                out[f"{tag}_rand{lvl}_{n_}"] = c
    real_encoder(ns, out)
    out = {k: (v.detach().cpu().numpy() if torch.is_tensor(v) else v) for k, v in out.items()}
    path = os.path.join(GOLD, "pixelnerf_reference_vectors.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
