"""Vanilla-NeRF training throughput on one GPU (BASELINE configs[0]): single-scene overfit of a 64 x 64 crop, 1024-ray batches,
NeRF(num_coarse_samples=64, num_fine_samples=64) = 65 + 129 points per ray, MSE of both levels (LitNeRF.training_step,
models/vanilla_nerf/model.py:273-299), Adam with the reference's learning-rate schedule (model.py:404-437, inlined below).

The step runs `NeRF.forward` under autograd (neo360_b200/vanilla.py: hand-written CUDA sampling, encodings and compositing forward and
backward, framework GEMMs for the dense layers).  The eager baseline is the same step through the oracle's stages
(oracle/vanilla_oracle.py: `vanilla_oracle.render`'s sampling, MLP and compositing, with the reference's detached level-0 weights,
helper.py:613) under autograd on the same GPU.

Prints one JSON line: training rays/s and ms per step from CUDA events after warm-up, the loss after the timed steps, the eager rate and
the speed-up over it, the whole-step FLOP rate (3 x 2 x 593 408 MAC per point x 194 points per ray: forward + two backward GEMMs of every
dense layer; a whole-step rate, not a kernel's share of peak), and the card name and power limit read in the same run.  Writes nothing.

    python tools/bench_vanilla_train.py [--steps 50] [--warmup 10] [--eager-steps 10] [--train-matmul fp32|tf32]
"""
import argparse
import json
import math
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F

from neo360_b200 import synth
from neo360_b200.vanilla import NeRF
from oracle import neo360_oracle as orc
from oracle import vanilla_oracle as vo

NC, NF, BATCH, CROP, FRAME = 64, 64, 1024, 64, 200
NEAR, FAR = 2.0, 6.0
MAC_PER_POINT = 63 * 256 + 4 * 256 * 256 + 319 * 256 + 2 * 256 * 256 + 256 * 256 + 256 + 283 * 128 + 128 * 3     # 593 408
POINTS_PER_RAY = (NC + 1) + (NC + 1 + NF)                                                                            # 194
LR_INIT, LR_FINAL, LR_DELAY_STEPS, LR_DELAY_MULT, MAX_STEPS = 5e-4, 5e-6, 2500, 0.01, 200000   # model.py:223-226


def learning_rate(step: int) -> float:
    """LitNeRF.optimizer_step (model.py:409-437): log-linear decay from lr_init to lr_final with a sine warm-up delay."""
    delay = LR_DELAY_MULT + (1 - LR_DELAY_MULT) * math.sin(0.5 * math.pi * min(max(step / LR_DELAY_STEPS, 0.0), 1.0))
    t = min(max(step / MAX_STEPS, 0.0), 1.0)
    return delay * math.exp(math.log(LR_INIT) * (1 - t) + math.log(LR_FINAL) * t)


def card(dev):
    name = torch.cuda.get_device_name(dev)
    try:
        import pynvml as nv
        nv.nvmlInit()
        h = nv.nvmlDeviceGetHandleByIndex(dev.index or 0)
        return name, nv.nvmlDeviceGetPowerManagementLimit(h) / 1000.0
    except Exception:
        pass
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", str(dev.index or 0)],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return name, float(out)
    except Exception:
        return name, None


def crop_batch(dev):
    """Rays and target colours of the central 64 x 64 crop of a seeded synthetic 200 x 200 frame (camera 4 units from the origin)."""
    pose = synth.look_at_pose(30.0, 1.0, 4.0)
    ro, vd, rd, _ = orc.rays_from_pose(orc.ray_directions(FRAME, FRAME, 1.1 * FRAME), pose[:3, :4])
    j, i = torch.meshgrid(torch.arange(CROP), torch.arange(CROP), indexing="ij")
    sel = ((j + (FRAME - CROP) // 2) * FRAME + i + (FRAME - CROP) // 2).reshape(-1)
    g = torch.Generator().manual_seed(0)
    img = F.interpolate(torch.rand(1, 3, 8, 8, generator=g), size=(CROP, CROP), mode="bilinear", align_corners=True)[0]
    target = img.permute(1, 2, 0).reshape(-1, 3)
    return {"rays_o": ro[sel].to(dev), "rays_d": rd[sel].to(dev), "viewdirs": vd[sel].to(dev)}, target.to(dev)


def eager_render(rays, P, randomized):
    o, d, vd = rays["rays_o"], rays["rays_d"], rays["viewdirs"]
    n = o.shape[0]
    denc = orc.pos_enc(vd, 0, 4)
    ret, t, w = [], None, None
    for lvl in range(2):
        if lvl == 0:
            t, pts = vo.sample_along_rays(o, vd, NC, NEAR, FAR, torch.rand(n, NC + 1, device=o.device) if randomized else None)
        else:
            t, pts = vo.sample_pdf(o, vd, t, w.detach(), NF, torch.rand(n, NF, device=o.device) if randomized else None)
        raw_rgb, raw_sigma = vo.mlp_forward(P, "coarse_mlp." if lvl == 0 else "fine_mlp.", orc.pos_enc(pts, 0, 10), denc)
        rgb = torch.sigmoid(raw_rgb) * (1 + 2 * 0.001) - 0.001
        comp, acc, w, depth = vo.composite(rgb, F.softplus(raw_sigma - 1.0), t, d, True)
        ret.append((comp, acc, depth))
    return ret


def timed(step, steps, warmup):
    for s in range(warmup):
        step(s)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for s in range(warmup, warmup + steps):
        step(s)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--eager-steps", type=int, default=10)
    ap.add_argument("--train-matmul", choices=["fp32", "tf32"], default="fp32")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_vanilla_train.py measures on a CUDA device; none is available")
    dev = torch.device("cuda:0")
    torch.backends.cuda.matmul.allow_tf32 = args.train_matmul == "tf32"
    rays, target = crop_batch(dev)
    P0 = synth.make_vanilla_params(0)
    gen = torch.Generator(device=dev).manual_seed(1)
    torch.manual_seed(0)

    net = NeRF(num_coarse_samples=NC, num_fine_samples=NF)
    net.load_state_dict(P0)
    net = net.to(dev).train()
    opt = torch.optim.Adam(net.parameters(), lr=LR_INIT, betas=(0.9, 0.999))
    state = {}

    def draw():
        idx = torch.randint(0, CROP * CROP, (BATCH,), device=dev, generator=gen)
        return {k: v[idx] for k, v in rays.items()}, target[idx]

    def step(s):
        batch, tgt = draw()
        ret = net(batch, True, True, NEAR, FAR)
        loss = F.mse_loss(ret[0][0], tgt) + F.mse_loss(ret[1][0], tgt)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        for pg in opt.param_groups:
            pg["lr"] = learning_rate(s)
        opt.step()
        state["loss"] = loss.detach()

    ms = timed(step, args.steps, args.warmup)
    loss = float(state["loss"])

    Pe = {k: v.to(dev).requires_grad_(True) for k, v in P0.items()}
    opt_e = torch.optim.Adam(list(Pe.values()), lr=LR_INIT, betas=(0.9, 0.999))

    def step_eager(s):
        batch, tgt = draw()
        ret = eager_render(batch, Pe, True)
        loss_e = F.mse_loss(ret[0][0], tgt) + F.mse_loss(ret[1][0], tgt)
        opt_e.zero_grad(set_to_none=True)
        loss_e.backward()
        for pg in opt_e.param_groups:
            pg["lr"] = learning_rate(s)
        opt_e.step()

    ms_eager = timed(step_eager, args.eager_steps, 2)
    name, power = card(dev)
    flop_ray = 3 * 2 * MAC_PER_POINT * POINTS_PER_RAY
    print(json.dumps(dict(
        metric="training rays/sec, vanilla NeRF single-scene overfit (BASELINE configs[0]), 1024-ray batches, 64+64 samples",
        value=BATCH / (ms * 1e-3), unit="rays/s", ms_per_step=ms, steps=args.steps, warmup=args.warmup, final_loss=loss,
        eager={"value": BATCH / (ms_eager * 1e-3), "ms_per_step": ms_eager, "steps": args.eager_steps,
               "what": "vanilla_oracle stages under autograd (detached level-0 weights), same GPU"},
        speedup_vs_eager=ms_eager / ms,
        whole_step_tflops=flop_ray * BATCH / (ms * 1e-3) / 1e12, flop_per_ray=flop_ray,
        flop_note="3 x 2 x 593408 MAC per point x 194 points per ray over the whole step time: a whole-step rate, not a kernel's share of peak",
        dtype=args.train_matmul, points_per_ray=POINTS_PER_RAY, gpu=name, power_limit_w=power,
        config={"crop": f"{CROP}x{CROP} of a seeded synthetic {FRAME}x{FRAME} frame", "near_far": [NEAR, FAR], "white_bkgd": True,
                "optimizer": "Adam(0.9, 0.999), lr schedule of model.py:409-437 (5e-4 -> 5e-6 over 200000 steps, delay 2500 x 0.01)",
                "hand_written": "sampling, inverse-CDF resampling, encodings, compositing forward and backward",
                "library": "dense layers (F.linear under autograd), activations, loss, Adam"})))


if __name__ == "__main__":
    main()
