"""TEST INFRASTRUCTURE ONLY -- golden vectors for vanilla NeRF's ray and pose gradients, from the UNMODIFIED reference NeRF module.

Run in the build container (where /root/reference exists):   python oracle/make_golden_camera_grad.py
Writes tests/golden/camera_grad_vectors.npz.  The reference NeRF (models/vanilla_nerf/model.py) runs in float64 under autograd on seeded
weights (synth.make_vanilla_params) and the rays of seeded pixels of a target pose; the loss is a seeded linear functional of both levels'
comp_rgb and acc.  Two cases:
  * "rays": rays_o, rays_d (scaled per ray, |rays_d| != 1 as the dataset hands them over, quirk Q15) and viewdirs are leaves: outputs and
    their gradients;
  * "pose": c2w (3,4) is the leaf; rays come from `camera_grad_model.rays_from_pose` (the reference's get_rays arithmetic out of place:
    its in-place normalisation is refused by autograd) of `get_ray_directions` pixels: the loss's gradient w.r.t. c2w.
  * "mip": the reference MipNeRF360 (models/mipnerf360/model.py) with rays_o, rays_d (scaled per ray), viewdirs and radii as leaves; the
    loss is a seeded linear functional of the NeRF level's rgb and every level's weights.
All deterministic (randomized=False); vanilla with a white background."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_shim  # noqa: E402
from oracle import camera_grad_model as cgm  # noqa: E402
from neo360_b200 import synth  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
W, H, B, NC, NF, SEED = 64, 48, 96, 16, 8, 0
NEAR, FAR = 0.2, 3.0
MIP_NP, MIP_NN, MIP_NEAR, MIP_FAR = 16, 8, 0.2, 6.0


def loss_of(ret, G):
    return sum((ret[l][0] * G[f"g_rgb{l}"]).sum() + (ret[l][1] * G[f"g_acc{l}"]).sum() for l in range(2))


def main():
    ns = ref_shim.load()
    focal = 0.8 * W
    dirs = ns.ray_utils.get_ray_directions(H, W, focal).double().reshape(-1, 3)
    assert torch.equal(dirs, cgm.camera_dirs(H, W, focal)), "camera_dirs differs from the reference's get_ray_directions"
    P = synth.make_vanilla_params(SEED)                 # drawn in float32 (the seeded draws depend on the default dtype)
    PM = synth.make_mip_params(SEED)
    ro32, vd32, rd32, rad32 = ns.ray_utils.get_rays(ns.ray_utils.get_ray_directions(H, W, focal), synth.target_pose(9, 100)[:3, :4],
                                                    output_view_dirs=True, output_radii=True)
    torch.set_default_dtype(torch.float64)
    net = ns.van_model.NeRF(num_coarse_samples=NC, num_fine_samples=NF).eval()
    net.load_state_dict(P, strict=True)
    net = net.double()
    for p in net.parameters():
        p.requires_grad_(False)
    pose = synth.target_pose(5, 100)[:3, :4].double()
    g = torch.Generator().manual_seed(60)
    sel = torch.randperm(H * W, generator=g)[:B]
    G = {f"g_{k}{l}": torch.randn(*((B, 3) if k == "rgb" else (B,)), generator=g, dtype=torch.float64) for l in range(2) for k in ("rgb", "acc")}
    out = {"cfg": np.array([W, H, B, NC, NF, SEED]), "near_far": np.array([NEAR, FAR]), "focal": np.array(focal), "pose": pose, "sel": sel}
    out.update(G)
    # case "rays"
    ro, vd, rd = cgm.rays_from_pose(dirs, pose)
    scale = 0.5 + torch.rand(B, 1, generator=g, dtype=torch.float64)
    rays = {"rays_o": ro[sel].clone().requires_grad_(True), "rays_d": (rd[sel] * scale).requires_grad_(True),
            "viewdirs": vd[sel].clone().requires_grad_(True)}
    ret = net(rays, False, True, NEAR, FAR)
    loss_of(ret, G).backward()
    for k in ("rays_o", "rays_d", "viewdirs"):
        out[f"rays_{k}"] = rays[k].detach()
        out[f"rays_g_{k}"] = rays[k].grad
    for l in range(2):
        out[f"rays_rgb{l}"], out[f"rays_acc{l}"] = ret[l][0].detach(), ret[l][1].detach()
    # case "pose"
    c2w = pose.clone().requires_grad_(True)
    ro, vd, rd = cgm.rays_from_pose(dirs, c2w)
    ret = net({"rays_o": ro[sel], "rays_d": rd[sel], "viewdirs": vd[sel]}, False, True, NEAR, FAR)
    loss_of(ret, G).backward()
    out["pose_g_c2w"] = c2w.grad
    for l in range(2):
        out[f"pose_rgb{l}"] = ret[l][0].detach()
    print("pose g_c2w", c2w.grad)
    # case "mip": the reference MipNeRF360 with every ray tensor a leaf; its contract detaches the Gaussians, so rays_o and radii get no
    # gradient and rays_d only through |rays_d| in the compositing
    mnet = ns.mip_model.MipNeRF360(num_prop_samples=MIP_NP, num_nerf_samples=MIP_NN).eval()
    mnet.load_state_dict(PM, strict=True)
    mnet = mnet.double()
    for p in mnet.parameters():
        p.requires_grad_(False)
    msel = torch.randperm(H * W, generator=g)[:B]
    mscale = 0.5 + torch.rand(B, 1, generator=g, dtype=torch.float64)
    mb = {"rays_o": ro32[msel].double(), "rays_d": rd32[msel].double() * mscale, "viewdirs": vd32[msel].double(),
          "radii": rad32[msel].double().reshape(-1, 1)}
    mb = {k: v.clone().requires_grad_(True) for k, v in mb.items()}
    GM = {"mip_g_rgb": torch.randn(B, 3, generator=g, dtype=torch.float64)}
    GM.update({f"mip_g_w{l}": torch.randn(B, (MIP_NP, MIP_NP, MIP_NN)[l], generator=g, dtype=torch.float64) for l in range(3)})
    ren, hist = mnet(mb, 1.0, False, False, MIP_NEAR, MIP_FAR)
    loss = (ren[2]["rgb"] * GM["mip_g_rgb"]).sum() + sum((hist[l]["weights"] * GM[f"mip_g_w{l}"]).sum() for l in range(3))
    loss.backward()
    out.update(GM)
    out["mip_cfg"] = np.array([MIP_NP, MIP_NN, MIP_NEAR, MIP_FAR])
    for k, v in mb.items():
        out[f"mip_{k}"] = v.detach()
        out[f"mip_g_{k}"] = v.grad if v.grad is not None else torch.zeros_like(v)
    out["mip_rgb2"] = ren[2]["rgb"].detach()
    print("mip grads None:", [k for k, v in mb.items() if v.grad is None])
    os.makedirs(GOLD, exist_ok=True)
    path = os.path.join(GOLD, "camera_grad_vectors.npz")
    np.savez_compressed(path, **{k: (v.numpy() if torch.is_tensor(v) else v) for k, v in out.items()})
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
