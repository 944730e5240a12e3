"""PixelNeRF throughput on one GPU: 640x480 frame rays/s of fp32 and tensor-core inference, and the step time of a 1024-ray training step (forward +
backward of both levels, encoder inside) with fp32 and with TF32 framework GEMMs, against the oracle's eager path on the same GPU.
Variants alternate in one process.  Prints one JSON line.

    python tools/bench_pixelnerf.py [--iters 5]"""
import argparse
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from neo360_b200 import PixelNeRF, synth  # noqa: E402
from oracle import neo360_oracle as orc, pixelnerf_oracle as por  # noqa: E402

NEAR, FAR = 0.02, 3.0


def timed(fn, iters):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_pixelnerf needs a GPU")
    dev = torch.device("cuda:0")
    W, H, nv = 640, 480, 3
    sc = synth.make_scene((W, H), nv, (8, 8), 0)
    net = PixelNeRF(num_src_views=nv)
    net.load_state_dict({**net.state_dict(), **synth.make_pixelnerf_params(0)})
    net = net.to(dev)
    ro, vd, rd, _ = orc.rays_from_pose(orc.ray_directions(H, W, 0.8 * W), synth.target_pose(3, 100)[:3, :4])
    imgs = torch.rand(nv, 3, H, W, generator=torch.Generator().manual_seed(0)).to(dev)
    src = {"src_imgs": imgs, "src_poses": sc["src_poses"].to(dev), "src_focal": sc["src_focal"].to(dev), "src_c": sc["src_c"].to(dev)}
    frame = {"rays_o": ro.to(dev), "rays_d": rd.to(dev), "viewdirs": vd.to(dev), **src}
    sel = torch.randperm(H * W, generator=torch.Generator().manual_seed(1))[:1024].to(dev)
    rays = {k: frame[k][sel] for k in ("rays_o", "rays_d", "viewdirs")}
    target = torch.rand(1024, 3, device=dev)

    def render(prec):
        net.eval()
        net.precision = prec
        with torch.no_grad():
            for i in range(0, H * W, 4096):          # the reference's chunked render loop; the encoder runs once (hoisted)
                net({**src, **{k: v[i:i + 4096] for k, v in frame.items() if k.startswith(("rays", "view"))}}, False, False, NEAR, FAR)

    def step_cuda():
        net.train()
        net.zero_grad(set_to_none=True)
        ret = net({**rays, **src}, True, False, NEAR, FAR)
        (((ret[0][0] - target) ** 2).mean() + ((ret[1][0] - target) ** 2).mean()).backward()

    P = {k: v.detach().clone().requires_grad_(True) for k, v in net.state_dict().items() if "mlp" in k}

    def step_eager():
        net.train()
        lat = net.encoder(imgs)
        osc = por.scene(lat, src["src_poses"], src["src_focal"].cpu(), src["src_c"].cpu(), (W, H))
        u = {"u0": torch.rand(1024, 65, device=dev), "u1": torch.rand(1024, 64, device=dev)}
        ret = por.render(rays, osc, P, 64, 64, NEAR, FAR, False, rand=u)
        (((ret[0][0] - target) ** 2).mean() + ((ret[1][0] - target) ** 2).mean()).backward()

    def with_tf32(flag, fn):
        def run():
            torch.backends.cuda.matmul.allow_tf32 = flag
            torch.backends.cudnn.allow_tf32 = flag
            fn()
        return run

    variants = {"render_fp32": lambda: render("fp32"), "render_tc": lambda: render("tc"), "train_fp32": with_tf32(False, step_cuda), "train_tf32": with_tf32(True, step_cuda),
                "train_eager_fp32": with_tf32(False, step_eager), "train_eager_tf32": with_tf32(True, step_eager)}
    for fn in variants.values():
        fn()
    res = {k: [] for k in variants}
    for _ in range(3):
        for k, fn in variants.items():
            res[k].append(timed(fn, args.iters))
    best = {k: min(v) for k, v in res.items()}
    q = torch.cuda.get_device_properties(0).name
    try:
        import subprocess
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except OSError:
        power = "unknown"
    print(json.dumps({"gpu": q, "power_limit": power, "frame_rays_per_s_fp32": round(H * W / best["render_fp32"]),
                      "frame_rays_per_s_tc": round(H * W / best["render_tc"]),
                      **{f"{k}_step_ms": round(1e3 * v, 2) for k, v in best.items() if k.startswith("train")}}))


if __name__ == "__main__":
    main()
