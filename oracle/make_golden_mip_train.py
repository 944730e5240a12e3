"""TEST INFRASTRUCTURE ONLY -- pins the Mip-NeRF 360 training loss and its gradients (LitMipNeRF360.training_step,
models/mipnerf360/model.py:427-456) of the UNMODIFIED reference, and checks that `mip_train_oracle` reproduces them.

For two cases (16/8 samples on 40 rays, 32/16 on 96 rays; rays of a turntable target view, injected jitter, train_frac 0.5, near / far
0.2 / 6) it runs the reference's MipNeRF360 in train mode under autograd, builds the loss from `LitMipNeRF360.interlevel_loss` /
`distortion_loss` (called unbound: both read only `ray_history`) and back-propagates.  The same step through `mip_train_oracle.render` +
`mip_train_oracle.training_loss_terms` must give the same loss terms and gradients (asserted; the measured difference is printed).  Writes
tests/golden/mip360_train_vectors.npz: the inputs, the three loss terms, each parameter's gradient norm and <g_p, r_p> for r_p drawn from a
seeded generator in state-dict order (full gradients are not stored: the NeRF MLP alone has about 9 M parameters).

    python oracle/make_golden_mip_train.py
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from neo360_b200 import synth
from neo360_b200.mip_basis import POS_BASIS_T
from oracle import mip_train_oracle as mto
from oracle import ref_shim
from oracle.make_golden import GOLD, RandQueue

CASES = {"t_tiny": (64, 48, 40, 16, 8, 0), "t_small": (64, 48, 96, 32, 16, 1)}
NEAR, FAR, TRAIN_FRAC = 0.2, 6.0, 0.5


def case_inputs(ns, W, H, B, seed):
    """B rays of target view 9 (the eval golden's camera, reference get_rays), the three (B,1) jitters and a target colour per ray."""
    pose = synth.target_pose(9, 100)
    dirs = ns.ray_utils.get_ray_directions(H, W, 0.8 * W)
    ro, vd, rd, radii = ns.ray_utils.get_rays(dirs, pose[:3, :4], output_view_dirs=True, output_radii=True)
    g = torch.Generator().manual_seed(170 + seed)
    sel = torch.randperm(H * W, generator=g)[:B]
    batch = {"rays_o": ro[sel].contiguous(), "rays_d": rd[sel].contiguous(), "viewdirs": vd[sel].contiguous(),
             "radii": radii[sel].reshape(-1, 1).contiguous()}
    jit = [torch.rand(B, 1, generator=g) for _ in range(3)]
    target = torch.rand(B, 3, generator=g)
    return batch, jit, target


def probes(params, seed):
    """r_p for every parameter, in the given (state-dict) order, from one seeded generator."""
    g = torch.Generator().manual_seed(1000 + seed)
    return {k: torch.randn(v.shape, generator=g, dtype=torch.float64) for k, v in params}


def oracle_step(batch, P, npp, nn_, jit, target, dtype=torch.float32):
    """Loss terms and gradients of the oracle's training step (float32 or float64 of the same inputs)."""
    b = {k: v.to(dtype) for k, v in batch.items()}
    Pg = {k: v.to(dtype).clone().requires_grad_(not k.endswith("pos_basis_t")) for k, v in P.items()}
    ren, hist = mto.render(b, Pg, POS_BASIS_T.to(dtype), npp, nn_, NEAR, FAR, TRAIN_FRAC, rand=[j.to(dtype) for j in jit])
    data, inter, dist = mto.training_loss_terms(ren, hist, target.to(dtype))
    (data + inter + 0.01 * dist).backward()
    return (data, inter, dist), {k: v.grad for k, v in Pg.items() if v.grad is not None}


def main():
    ns = ref_shim.load()
    out = {}
    for tag, (W, H, B, npp, nn_, seed) in CASES.items():
        P = synth.make_mip_params(seed)
        net = ns.mip_model.MipNeRF360(num_prop_samples=npp, num_nerf_samples=nn_).train()
        net.load_state_dict(P, strict=True)
        batch, jit, target = case_inputs(ns, W, H, B, seed)
        with RandQueue(jit):
            ren, hist = net(batch, TRAIN_FRAC, True, True, NEAR, FAR)
        Lm = ns.mip_model.LitMipNeRF360
        data = torch.sqrt(ns.mip_helper.img2mse(ren[-1]["rgb"], target) + 0.001 ** 2)
        inter, dist = Lm.interlevel_loss(None, hist), Lm.distortion_loss(None, hist)
        (data + inter + 0.01 * dist).backward()
        gref = {k: p.grad for k, p in net.named_parameters()}
        assert all(g is not None for g in gref.values()), [k for k, g in gref.items() if g is None]
        (o_data, o_inter, o_dist), gorc = oracle_step(batch, P, npp, nn_, jit, target)
        assert set(gorc) == set(gref), set(gorc) ^ set(gref)
        dl = max(abs(float(a.detach()) - float(b.detach())) for a, b in ((o_data, data), (o_inter, inter), (o_dist, dist)))
        dg = max(float((gorc[k] - gref[k]).abs().max()) / max(float(gref[k].abs().max()), 1e-30) for k in gref)
        print(f"{tag}: oracle vs reference: loss terms max|diff| {dl:.3e}, gradients max|diff| / max|g| {dg:.3e}")
        assert dl < 1e-5 and dg < 1e-3, (dl, dg)
        names = list(gref)
        r = probes([(k, gref[k]) for k in names], seed)
        out.update({f"{tag}_cfg": np.array([W, H, B, npp, nn_, seed]), f"{tag}_near_far_frac": np.array([NEAR, FAR, TRAIN_FRAC]),
                    f"{tag}_target": target, f"{tag}_loss": torch.stack([data, inter, dist]).detach(),
                    f"{tag}_names": np.array(names), f"{tag}_gnorm": torch.stack([gref[k].double().norm() for k in names]),
                    f"{tag}_gdot": torch.stack([(gref[k].double() * r[k]).sum() for k in names])})
        for k, v in batch.items():
            out[f"{tag}_{k}"] = v
        for i in range(3):
            out[f"{tag}_jit{i}"] = jit[i]
    path = os.path.join(GOLD, "mip360_train_vectors.npz")
    np.savez_compressed(path, **{k: (v.detach().numpy() if torch.is_tensor(v) else v) for k, v in out.items()})
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
