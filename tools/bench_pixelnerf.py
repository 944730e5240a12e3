"""PixelNeRF throughput on one GPU: 640x480 frame rays/s of fp32 and tensor-core inference, and the step time of a 1024-ray training step (forward +
backward of both levels, encoder inside) with fp32 and with TF32 framework GEMMs, with the framework MLP under torch.autocast(bfloat16)
(TF32 allowed elsewhere), and with train_precision="tc" (trunk on the tensor cores in bf16; encoder, projection and head framework ops with
TF32 allowed), against the oracle's eager path on the same GPU.  Variants alternate in one process.  For each CUDA training variant it also
prints the step's split by CUDA events (encoder forward + backward against the rest), its peak memory, and the projection GEMM of the "tc"
path (P0 = latent . W0[:, 63:575]^T, forward + backward, one level) timed alone.  Prints one JSON line.

    python tools/bench_pixelnerf.py [--iters 5]"""
import argparse
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from neo360_b200 import PixelNeRF, pixelnerf, synth  # noqa: E402
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

    def step_cuda(tprec="fp32"):
        net.train()
        net.train_precision = tprec
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

    mlp_train = pixelnerf._mlp_train

    def step_autocast():
        def mlp_autocast(*a):
            with torch.autocast("cuda", dtype=torch.bfloat16):
                return tuple(t.float() for t in mlp_train(*a))
        pixelnerf._mlp_train = mlp_autocast
        try:
            step_cuda()
        finally:
            pixelnerf._mlp_train = mlp_train

    lat_shape = net.encoder(imgs).shape
    lat_p = torch.randn(lat_shape[0], lat_shape[2], lat_shape[3], lat_shape[1], device=dev, requires_grad=True)
    w0 = net.coarse_mlp.pts_linears[0].weight

    def projection():
        lat_p.grad = None
        w0.grad = None
        p0 = lat_p @ w0[:, 63:].t()
        p0.backward(torch.ones_like(p0))

    def split(fn):
        """(encoder forward + backward ms, rest ms) of one step by CUDA events: the encoder's backward runs from the moment the latent's
        gradient is complete to the end of the step (its inputs are leaves)."""
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
        enc_forward = net.encoder.forward

        def forward(x):
            ev[1].record()
            lat = enc_forward(x)
            ev[2].record()
            lat.register_hook(lambda g: ev[3].record())
            return lat

        net.encoder.forward = forward
        try:
            torch.cuda.synchronize()
            ev[0].record()
            fn()
            ev[4].record()
        finally:
            del net.encoder.forward
        torch.cuda.synchronize()
        total = ev[0].elapsed_time(ev[4])
        enc = ev[1].elapsed_time(ev[2]) + ev[3].elapsed_time(ev[4])
        return round(enc, 2), round(total - enc, 2)

    def with_tf32(flag, fn):
        def run():
            torch.backends.cuda.matmul.allow_tf32 = flag
            torch.backends.cudnn.allow_tf32 = flag
            fn()
        return run

    variants = {"render_fp32": lambda: render("fp32"), "render_tc": lambda: render("tc"), "train_fp32": with_tf32(False, step_cuda), "train_tf32": with_tf32(True, step_cuda),
                "train_autocast": with_tf32(True, step_autocast), "train_tc": with_tf32(True, lambda: step_cuda("tc")),
                "train_eager_fp32": with_tf32(False, step_eager), "train_eager_tf32": with_tf32(True, step_eager)}
    variants["projection_tf32"] = with_tf32(True, projection)
    for fn in variants.values():
        fn()
    res = {k: [] for k in variants}
    peak = {}
    for _ in range(3):
        for k, fn in variants.items():
            torch.cuda.reset_peak_memory_stats()
            res[k].append(timed(fn, args.iters))
            peak[k] = max(peak.get(k, 0), torch.cuda.max_memory_allocated())
    best = {k: min(v) for k, v in res.items()}
    cuda_train = ("train_fp32", "train_tf32", "train_autocast", "train_tc")
    splits = {k: [split(variants[k]) for _ in range(3)] for k in cuda_train}
    q = torch.cuda.get_device_properties(0).name
    try:
        import subprocess
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except OSError:
        power = "unknown"
    print(json.dumps({"gpu": q, "power_limit": power, "frame_rays_per_s_fp32": round(H * W / best["render_fp32"]),
                      "frame_rays_per_s_tc": round(H * W / best["render_tc"]),
                      **{f"{k}_step_ms": round(1e3 * v, 2) for k, v in best.items() if k.startswith("train")},
                      "projection_fwd_bwd_ms_per_level": round(1e3 * best["projection_tf32"], 3),
                      "split_encoder_vs_rest_ms": {k: min(v, key=sum) for k, v in splits.items()},
                      "peak_mem_gib": {k: round(peak[k] / 2 ** 30, 2) for k in variants if k.startswith("train")}}))


if __name__ == "__main__":
    main()
