"""Refine noisy camera poses of vanilla NeRF by photometric gradient (BARF / NeRF-- style), on a seeded synthetic model.

    python tools/refine_poses.py --model vanilla [--steps 200] [--time]

1. renders each level's target images from seeded NeRF weights (synth.make_vanilla_params) at ground-truth turntable poses;
2. perturbs the poses (a rotation of --rot-deg degrees and a translation of --trans about random axes, per view);
3. freezes the MLPs;
4. optimises a `cameras.PoseCorrection` with Adam on the MSE of both levels, rays from `ops.sample_rays` on the corrected poses;
5. prints the mean rotation (degrees) and translation errors per step.

--time reports, on the GPU, ms per training step of vanilla NeRF at BASELINE configs[0] (1024-ray batches, 64 + 64 samples) with the
MLP training, with and without ray gradients (rays from sample_rays on poses that require grad, vs. plain rays), for train_precision
fp32 and tc, the two variants alternated in one process, with the card name and power limit.
Only vanilla NeRF: Mip-NeRF 360's reference detaches the contracted Gaussians (models/mipnerf360/helper.py:63-66), so its rays_o gets no
gradient and a pose correction through it reaches the rotation only."""
import argparse
import math
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from neo360_b200 import ops, synth  # noqa: E402
from neo360_b200.cameras import PoseCorrection, so3_exp  # noqa: E402
from neo360_b200.vanilla import NeRF  # noqa: E402

NEAR, FAR = 0.2, 3.0


def _net(nc, nf, prec, dev, seed=0):
    net = NeRF(num_coarse_samples=nc, num_fine_samples=nf, train_precision=prec)
    net.load_state_dict(synth.make_vanilla_params(seed))
    return net.to(dev)


def pose_errors(est, gt):
    """Mean rotation angle (degrees) of R_gt^T R_est and mean |t_est - t_gt| over the views, in float64 (acos of the trace in fp32
    cannot resolve angles below about 0.02 degrees)."""
    est, gt = est.double(), gt.double()
    Rr = gt[:, :3, :3].transpose(1, 2) @ est[:, :3, :3]
    cos = ((Rr.diagonal(dim1=1, dim2=2).sum(-1) - 1) / 2).clamp(-1, 1)
    return float(torch.rad2deg(torch.acos(cos)).mean()), float((est[:, :3, 3] - gt[:, :3, 3]).norm(dim=-1).mean())


def refine(steps=200, n_views=4, H=32, W=32, nc=32, nf=32, rot_deg=1.0, trans=0.02, lr=1e-3, seed=0, dev="cuda", log=None):
    """Returns the (rotation, translation) errors before and after `steps` Adam steps on the MSE over every pixel of the views."""
    dev = torch.device(dev)
    g = torch.Generator().manual_seed(100 + seed)
    gt = torch.stack([synth.target_pose(25 * k + 3, 100)[:3, :4] for k in range(n_views)]).to(dev)
    focal = 0.8 * W
    net = _net(nc, nf, "fp32", dev, seed).eval().requires_grad_(False)
    with torch.no_grad():
        pix = torch.arange(n_views * H * W, device=dev)
        o, vd, rd, _, _ = ops.sample_rays(pix, H, W, focal, gt)
        target = [r[0] for r in net({"rays_o": o, "rays_d": rd, "viewdirs": vd}, False, True, NEAR, FAR)]      # each level's image
    axis = lambda: torch.nn.functional.normalize(torch.randn(n_views, 3, generator=g, dtype=torch.float64), dim=-1)
    dR = so3_exp(axis() * math.radians(rot_deg)).float().to(dev)
    noisy = torch.cat([gt[:, :, :3] @ dR, gt[:, :, 3:] + (axis() * trans).float().to(dev)[..., None]], -1)
    pc = PoseCorrection(n_views).to(dev)
    opt = torch.optim.Adam(pc.parameters(), lr=lr)
    before = pose_errors(noisy, gt)
    for s in range(steps):
        o, vd, rd, _, _ = ops.sample_rays(pix, H, W, focal, pc(noisy))
        ret = net({"rays_o": o, "rays_d": rd, "viewdirs": vd}, False, True, NEAR, FAR)
        loss = sum(((r[0] - tg) ** 2).mean() for r, tg in zip(ret, target))
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
        if log is not None and (s % 10 == 0 or s == steps - 1):
            with torch.no_grad():
                e = pose_errors(pc(noisy), gt)
            log(f"step {s:4d}  loss {float(loss.detach()):.3e}  rotation {e[0]:.4f} deg  translation {e[1]:.5f}")
    with torch.no_grad():
        after = pose_errors(pc(noisy), gt)
    return before, after


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def time_steps(steps=50, warmup=10, rounds=3):
    """ms per training step (MLP parameters train) with and without ray gradients, BASELINE configs[0]; variants alternated."""
    dev = torch.device("cuda")
    H = W = 64
    T, focal, nc, nf, batch = 4, 0.8 * 64, 64, 64, 1024
    poses = torch.stack([synth.target_pose(25 * k, 100)[:3, :4] for k in range(T)]).to(dev)
    target = torch.rand(T * H * W, 3, device=dev)
    res = {}
    for prec in ("fp32", "tc"):
        net = _net(nc, nf, prec, dev).train()
        opt = torch.optim.Adam(net.parameters(), lr=5e-4)
        pc = PoseCorrection(T).to(dev)
        popt = torch.optim.Adam(pc.parameters(), lr=1e-3)
        g = torch.Generator(device=dev).manual_seed(0)

        def step(ray_grad):
            sel = torch.randint(0, T * H * W, (batch,), device=dev, generator=g)
            c2w = pc(poses) if ray_grad else poses
            o, vd, rd, _, _ = ops.sample_rays(sel, H, W, focal, c2w)
            ret = net({"rays_o": o, "rays_d": rd, "viewdirs": vd}, True, True, NEAR, FAR)
            loss = sum(((r[0] - target[sel]) ** 2).mean() for r in ret)
            opt.zero_grad(set_to_none=True)
            popt.zero_grad(set_to_none=True)
            loss.backward()
            opt.step()
            if ray_grad:
                popt.step()

        for v in (False, True):
            for _ in range(warmup):
                step(v)
        times = {False: [], True: []}
        for _ in range(rounds):
            for v in (False, True):
                torch.cuda.synchronize()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(steps):
                    step(v)
                b.record()
                torch.cuda.synchronize()
                times[v].append(a.elapsed_time(b) / steps)
        res[prec] = {"without_ray_grad_ms": min(times[False]), "with_ray_grad_ms": min(times[True]),
                     "spread_ms": [max(times[False]) - min(times[False]), max(times[True]) - min(times[True])]}
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--model", choices=["vanilla"], default="vanilla")
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--rot-deg", type=float, default=1.0)
    ap.add_argument("--trans", type=float, default=0.02)
    ap.add_argument("--time", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("refine_poses.py needs a CUDA device")
    from neo360_b200 import build
    build.build()
    before, after = refine(a.steps, rot_deg=a.rot_deg, trans=a.trans, log=print)
    print(f"rotation error {before[0]:.4f} -> {after[0]:.4f} deg, translation error {before[1]:.5f} -> {after[1]:.5f}")
    if a.time:
        print("card:", card())
        for prec, r in time_steps().items():
            print(f"vanilla BASELINE configs[0] train_precision={prec}: {r['without_ray_grad_ms']:.3f} ms/step without ray gradients, "
                  f"{r['with_ray_grad_ms']:.3f} ms/step with (spread over rounds {r['spread_ms'][0]:.3f} / {r['spread_ms'][1]:.3f} ms)")


if __name__ == "__main__":
    main()
