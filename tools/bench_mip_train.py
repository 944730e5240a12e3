"""Mip-NeRF 360 training throughput on one GPU: 2048-ray batches (LitMipNeRF360.train_dataloader, models/mipnerf360/model.py:629-636),
MipNeRF360(num_prop_samples=64, num_nerf_samples=32) (the reference defaults: 64 + 64 proposal and 32 NeRF samples per ray), near / far
0.2 / 100 as `bench.py --mode mip360`, the reference's training loss (LitMipNeRF360.training_step, model.py:427-456: Charbonnier data term,
interlevel loss, 0.01 x distortion loss) and Adam with its learning-rate schedule (model.py:372-376, 599-627, inlined below:
2e-3 -> 2e-5 over 1e6 steps, delay 512 x 0.01) and train_frac = step / 1e6.

The step runs `MipNeRF360.forward` under autograd (neo360_b200/mip.py: hand-written CUDA resampling, IPE features, compositing forward and
backward; framework GEMMs for the dense layers).  Rays are drawn from 640 x 480 frames of synthetic poses (`ops.get_rays`), with fixed
random target colours.  The eager baseline is the same step through `mip_train_oracle.render` (the reference formulation on `mip_oracle`'s
stages, sdist detached) and `mip_train_oracle`'s loss under autograd on the same GPU.

Prints one JSON line: training rays/s and ms per step from CUDA events after warm-up, the loss after the timed steps, the eager rate and the
speed-up over it, the whole-step FLOP rate (3 x 2 x 319 217 664 MAC per ray: forward + two backward GEMMs of every dense layer; a whole-step
rate, not a kernel's share of peak), and the card name and power limit read in the same run.  Writes nothing.

    python tools/bench_mip_train.py [--steps 20] [--warmup 5] [--eager-steps 5] [--train-matmul fp32|tf32]
"""
import argparse
import json
import math
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from neo360_b200 import ops, synth
from neo360_b200.mip import MipNeRF360, training_loss
from neo360_b200.mip_basis import POS_BASIS_T
from oracle import mip_train_oracle as mto
from tools.bench_vanilla_train import card, timed

NP, NN, BATCH, W, H, FRAMES = 64, 32, 2048, 640, 480, 8
NEAR, FAR = 0.2, 100.0
MAC_PER_RAY = 2 * NP * 325888 + NN * 8672000                     # 319 217 664: two 4 x 256 PropMLPs, one 8 x 1024 NeRFMLP (+ rgb head)
LR_INIT, LR_FINAL, LR_DELAY_STEPS, LR_DELAY_MULT, MAX_STEPS = 2e-3, 2e-5, 512, 0.01, 1000000


def learning_rate(step: int) -> float:
    """LitMipNeRF360.optimizer_step (model.py:599-627): log-linear decay with a sine warm-up delay."""
    delay = LR_DELAY_MULT + (1 - LR_DELAY_MULT) * math.sin(0.5 * math.pi * min(max(step / LR_DELAY_STEPS, 0.0), 1.0))
    t = min(max(step / MAX_STEPS, 0.0), 1.0)
    return delay * math.exp(math.log(LR_INIT) * (1 - t) + math.log(LR_FINAL) * t)


def ray_pool(dev):
    """Rays of FRAMES 640 x 480 views (ops.get_rays, focal 0.8 W) of the synthetic turntable, and a fixed random target colour per ray."""
    parts = {k: [] for k in ("rays_o", "viewdirs", "rays_d", "radii")}
    for f in range(FRAMES):
        c2w = synth.target_pose(7 * f, 100)[:3, :4].float().to(dev)
        for k, v in zip(parts, ops.get_rays(H, W, 0.8 * W, c2w)):
            parts[k].append(v.reshape(v.shape[0], -1))
    rays = {k: torch.cat(v) for k, v in parts.items()}
    target = torch.rand(rays["rays_o"].shape[0], 3, generator=torch.Generator().manual_seed(0)).to(dev)
    return rays, target


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--eager-steps", type=int, default=5)
    ap.add_argument("--train-matmul", choices=["fp32", "tf32"], default="fp32")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mip_train.py measures on a CUDA device; none is available")
    dev = torch.device("cuda:0")
    torch.backends.cuda.matmul.allow_tf32 = args.train_matmul == "tf32"
    rays, target = ray_pool(dev)
    P0 = synth.make_mip_params(0)
    gen = torch.Generator(device=dev).manual_seed(1)
    torch.manual_seed(0)

    net = MipNeRF360(num_prop_samples=NP, num_nerf_samples=NN)
    net.load_state_dict(P0)
    net = net.to(dev).train()
    params = [p for p in net.parameters() if p.requires_grad]
    opt = torch.optim.Adam(params, lr=LR_INIT, betas=(0.9, 0.999))
    state = {}

    def draw():
        idx = torch.randint(0, rays["rays_o"].shape[0], (BATCH,), device=dev, generator=gen)
        return {k: v[idx] for k, v in rays.items()}, target[idx]

    def step(s):
        batch, tgt = draw()
        ren, hist = net(batch, s / MAX_STEPS, True, True, NEAR, FAR)
        loss = training_loss(ren, hist, tgt)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        for pg in opt.param_groups:
            pg["lr"] = learning_rate(s)
        opt.step()
        state["loss"] = loss.detach()

    ms = timed(step, args.steps, args.warmup)
    loss = float(state["loss"])

    Pe = {k: v.to(dev).requires_grad_(not k.endswith("pos_basis_t")) for k, v in P0.items()}
    opt_e = torch.optim.Adam([v for v in Pe.values() if v.requires_grad], lr=LR_INIT, betas=(0.9, 0.999))
    basis = POS_BASIS_T.to(dev)

    def step_eager(s):
        batch, tgt = draw()
        jit = [torch.rand(BATCH, 1, device=dev) for _ in range(3)]
        ren, hist = mto.render(batch, Pe, basis, NP, NN, NEAR, FAR, s / MAX_STEPS, rand=jit)
        data, inter, dist = mto.training_loss_terms(ren, hist, tgt)
        loss_e = data + inter + 0.01 * dist
        opt_e.zero_grad(set_to_none=True)
        loss_e.backward()
        for pg in opt_e.param_groups:
            pg["lr"] = learning_rate(s)
        opt_e.step()

    ms_eager = timed(step_eager, args.eager_steps, 2)
    name, power = card(dev)
    flop_ray = 3 * 2 * MAC_PER_RAY
    print(json.dumps(dict(
        metric="training rays/sec, Mip-NeRF 360, 2048-ray batches, 64/64/32 samples",
        value=BATCH / (ms * 1e-3), unit="rays/s", ms_per_step=ms, steps=args.steps, warmup=args.warmup, final_loss=loss,
        eager={"value": BATCH / (ms_eager * 1e-3), "ms_per_step": ms_eager, "steps": args.eager_steps,
               "what": "mip_train_oracle.render + its loss under autograd (sdist detached), same GPU"},
        speedup_vs_eager=ms_eager / ms,
        whole_step_tflops=flop_ray * BATCH / (ms * 1e-3) / 1e12, flop_per_ray=flop_ray,
        flop_note="3 x 2 x 319217664 MAC per ray over the whole step time: a whole-step rate, not a kernel's share of peak",
        dtype=args.train_matmul, gpu=name, power_limit_w=power,
        config={"rays": f"{FRAMES} synthetic 640x480 frames (ops.get_rays), fixed random targets", "near_far": [NEAR, FAR],
                "optimizer": "Adam(0.9, 0.999), lr schedule of model.py:599-627 (2e-3 -> 2e-5 over 1e6 steps, delay 512 x 0.01), "
                             "train_frac = step / 1e6",
                "hand_written": "proposal resampling, IPE features, direction encoding, compositing forward and backward",
                "library": "dense layers (F.linear under autograd), activations inside the compositing kernel, losses, Adam"})))


if __name__ == "__main__":
    main()
