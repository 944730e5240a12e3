"""What torch.use_deterministic_algorithms(True) costs in the training step, on one GPU.

Step time with deterministic mode off and on, alternated in one run (rounds of --steps steps each, after --warmup steps of both), for:
  * NeO-360 BASELINE configs[3]: `training.bench_train`'s step itself (4096 rays, 128 + 64 samples, 3 source views, GridEncoder inside the
    step, projected formulation, Adam), with fp32 and with TF32 framework GEMMs / convolutions;
  * vanilla NeRF configs[0]: NeRF(64, 64), 1024 rays, MSE of both levels, Adam;
  * Mip-NeRF 360 64/64/32: 2048 rays, `mip.training_loss`, Adam.
And the kernel time of the lookup backward at the production shape (the projected maps' 256 channels, 3 views, 4096 x 257 lookup points of
one level): `neo_index_maps_bwd` (float4 atomics) against `neo_index_maps_bwd_det` (sort + segmented reduction), CUDA events over 20 calls.
Prints one JSON line with the card name and power limit read in the same run.  Writes nothing.

    CUBLAS_WORKSPACE_CONFIG=:4096:8 python tools/bench_deterministic_train.py [--steps 10] [--warmup 3] [--rounds 3]
"""
import argparse
import json
import os
import sys
import types

os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from neo360_b200 import _lib as L
from neo360_b200 import mip, ops, synth, training
from tools.bench_vanilla_train import card


def alternate(step, steps, warmup, rounds):
    """ms per step {False: flag off, True: flag on}: warm-up of both, then `rounds` alternating windows of `steps` steps."""
    ms = {False: [], True: []}
    s = 0
    for det in (False, True):
        torch.use_deterministic_algorithms(det)
        for _ in range(warmup):
            step(s)
            s += 1
    for _ in range(rounds):
        for det in (False, True):
            torch.use_deterministic_algorithms(det)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(steps):
                step(s)
                s += 1
            e1.record()
            torch.cuda.synchronize()
            ms[det].append(e0.elapsed_time(e1) / steps)
    torch.use_deterministic_algorithms(False)
    return {"off_ms": min(ms[False]), "on_ms": min(ms[True]), "on_over_off": min(ms[True]) / min(ms[False])}


def neo_step(dev, tf32, args):
    out = {}

    def timed(step, steps, warmup, dev_, dist):
        out.update(alternate(step, args.steps, args.warmup, args.rounds))
        return 1.0
    ns = types.SimpleNamespace(batch_rays=4096, freeze_encoder=False, train_matmul="tf32" if tf32 else "fp32", train_formulation="projected",
                               steps=args.steps, warmup=args.warmup)
    training.bench_train(ns, 0, 1, 0, dev, None, None, {}, None, timed)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    return out


def vanilla_step(dev, args):
    from neo360_b200.vanilla import NeRF
    torch.manual_seed(0)
    net = NeRF(num_coarse_samples=64, num_fine_samples=64)
    net.load_state_dict(synth.make_vanilla_params(0))
    net = net.to(dev).train()
    c2w = synth.target_pose(3, 100)[:3, :4].float().to(dev)
    o, vd, rd, _ = ops.get_rays(480, 640, 0.8 * 640, c2w)
    sel = torch.randperm(o.reshape(-1, 3).shape[0], generator=torch.Generator().manual_seed(0))[:1024].to(dev)
    rays = {"rays_o": o.reshape(-1, 3)[sel].contiguous(), "rays_d": rd.reshape(-1, 3)[sel].contiguous(), "viewdirs": vd.reshape(-1, 3)[sel].contiguous()}
    tgt = torch.rand(1024, 3, generator=torch.Generator().manual_seed(9)).to(dev)
    opt = torch.optim.Adam(net.parameters(), lr=5e-4)

    def step(s):
        ret = net(rays, True, False, 2.0, 6.0)
        loss = ((ret[0][0] - tgt) ** 2).mean() + ((ret[1][0] - tgt) ** 2).mean()
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
    return alternate(step, args.steps, args.warmup, args.rounds)


def mip_step(dev, args):
    from neo360_b200.mip import MipNeRF360
    torch.manual_seed(0)
    net = MipNeRF360(num_prop_samples=64, num_nerf_samples=32)
    net.load_state_dict(synth.make_mip_params(0))
    net = net.to(dev).train()
    c2w = synth.target_pose(7, 100)[:3, :4].float().to(dev)
    o, vd, rd, radii = ops.get_rays(480, 640, 0.8 * 640, c2w)
    sel = torch.randperm(o.reshape(-1, 3).shape[0], generator=torch.Generator().manual_seed(0))[:2048].to(dev)
    rays = {"rays_o": o.reshape(-1, 3)[sel].contiguous(), "rays_d": rd.reshape(-1, 3)[sel].contiguous(),
            "viewdirs": vd.reshape(-1, 3)[sel].contiguous(), "radii": radii.reshape(-1, 1)[sel].contiguous()}
    tgt = torch.rand(2048, 3, generator=torch.Generator().manual_seed(9)).to(dev)
    params = [p for p in net.parameters() if p.requires_grad]
    opt = torch.optim.Adam(params, lr=2e-3)

    def step(s):
        ren, hist = net(rays, 0.5, True, True, 0.2, 100.0)
        loss = mip.training_loss(ren, hist, tgt)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
    return alternate(step, args.steps, args.warmup, args.rounds)


def lookup_kernels(dev):
    """neo_index_maps_bwd against neo_index_maps_bwd_det: 3 views, C = 256, 4096 x 257 points inside the unit sphere."""
    from neo360_b200 import NeRF_TP
    nv, C, M = 3, 256, 4096 * 257
    sc = synth.make_scene((640, 480), nv, (120, 160), 0)
    net = NeRF_TP(num_coarse_samples=8, num_fine_samples=4, num_src_views=nv, precision="fp32").to(dev)
    net.set_scene(*[sc[k].to(dev) for k in ("planes_xz", "planes_xy", "planes_yz", "latent", "src_poses", "src_focal", "src_c")], sc["img_wh"],
                  precisions=[])
    h = net._scene.handle
    g = torch.Generator(device=dev).manual_seed(0)
    v = torch.randn(M, 3, generator=g, device=dev)
    pts = (v / v.norm(dim=-1, keepdim=True) * torch.rand(M, 1, generator=g, device=dev) ** (1 / 3)).contiguous()
    gl, gw = torch.randn(nv * M, C, generator=g, device=dev), torch.randn(nv * M, C, generator=g, device=dev)
    lat = torch.zeros(nv, 240, 320, C, device=dev)
    pl = [torch.zeros(nv, 120, 160, C, device=dev) for _ in range(3)]
    lib, P, s = L.load(), L.ptr, torch.cuda.current_stream().cuda_stream
    need = lib.neo_index_maps_bwd_det_workspace_bytes(h, M, C)
    ws = torch.empty(need, dtype=torch.uint8, device=dev)
    calls = {"atomic": lambda: lib.neo_index_maps_bwd(h, P(pts), M, C, P(gl), P(gw), P(lat), *[P(x) for x in pl], s),
             "det": lambda: lib.neo_index_maps_bwd_det(h, P(pts), M, C, P(gl), P(gw), P(lat), *[P(x) for x in pl], P(ws), need, s)}
    res = {}
    for name, fn in calls.items():
        for _ in range(3):
            L.check(fn())
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(20):
            L.check(fn())
        e1.record()
        torch.cuda.synchronize()
        res[name + "_ms"] = e0.elapsed_time(e1) / 20
    res["det_over_atomic"] = res["det_ms"] / res["atomic_ms"]
    res["workspace_bytes"] = need
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_deterministic_train.py measures on a CUDA device; none is available")
    dev = torch.device("cuda:0")
    torch.backends.cudnn.benchmark = False
    name, power = card(dev)
    out = {"card": name, "power_limit_w": power, "steps_per_window": args.steps, "rounds": args.rounds,
           "lookup_bwd_production_shape": lookup_kernels(dev),
           "neo360_configs3_fp32": neo_step(dev, False, args), "neo360_configs3_tf32": neo_step(dev, True, args),
           "vanilla_configs0": vanilla_step(dev, args), "mip360_64_64_32": mip_step(dev, args)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
