"""NeO-360 throughput against the number of source views: rendering and test-time optimisation at NV = 1, 3 and 5.

    python tools/bench_views.py                       # everything, one JSON line per measurement and a summary table
    python tools/bench_views.py --views 5 --skip-tto  # rendering only, 5 views

Rendering: `render_rays_test(chunk=1024)` of one turntable frame, 128 + 64 samples (the benchmark's), source images and latent of
640x480 or 320x240 (the reference's 5-view evaluation size), 120x160 tri-planes.  "tc" renders the whole frame in 8x4 pixel blocks;
"fp32" (the parity path, about 50x slower) renders the frame's first --fp32-rays rays.  Rays per second over device-synchronised calls,
median of --repeats after a warm-up.
Test-time optimisation: one `training.test_time_step` (500 rays of one source view, 128 + 256 samples as the reference's NeRF_TP
defaults, GridEncoder inside the step with the ResNet frozen, plain Adam) at 640x480 sources, with `train_precision` "fp32" and "tc",
with the frozen ResNet run once per scene ("hoisted", the library's behaviour) and, for comparison, once per step.  Median step time.
The card's name, power limit and SM clock limit are printed with the numbers.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def median_time(fn, repeats, warmup=1):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return sorted(ts)[len(ts) // 2]


def frame_rays(W, H, dev, view=7):
    from neo360_b200 import synth
    from oracle import neo360_oracle as orc
    pose = synth.target_pose(view, 100)
    ro, vd, rd, _ = orc.rays_from_pose(orc.ray_directions(H, W, 0.8 * W), pose[:3, :4])
    return {"rays_o": ro.to(dev), "rays_d": rd.to(dev), "viewdirs": vd.to(dev)}


def bench_render(dev, nv, W, H, precision, fp32_rays, repeats):
    from neo360_b200 import NeRF_TP, synth
    sc = synth.make_scene((W, H), nv, (120, 160), seed=0)
    net = NeRF_TP(num_coarse_samples=128, num_fine_samples=64, num_src_views=nv, precision=precision).eval()
    net.load_state_dict(synth.make_mlp_params(0))
    net = net.to(dev)
    net.set_scene(*[sc[k].to(dev) for k in ("planes_xz", "planes_xy", "planes_yz", "latent", "src_poses", "src_focal", "src_c")],
                  sc["img_wh"], precisions=[precision])
    rays = frame_rays(W, H, dev)
    if precision == "fp32":
        rays = {k: v[:fp32_rays].contiguous() for k, v in rays.items()}
        kw = {}
    else:
        kw = {"img_wh": (W, H)}
    n = rays["rays_o"].shape[0]
    with torch.no_grad():
        t = median_time(lambda: net.render_rays_test(rays, chunk=1024, **kw), repeats)
    net.check()
    return {"kind": "render", "views": nv, "size": f"{W}x{H}", "precision": precision, "rays": n, "s_per_call": t, "rays_per_s": n / t}


def bench_tto(dev, nv, train_precision, hoisted, repeats):
    from neo360_b200 import batches, training
    from optimize_source_views import make_setup
    torch.cuda.reset_peak_memory_stats()
    net, opt, views, src = make_setup(dev, nv, (640, 480), train_precision=train_precision)
    if not hoisted:
        net.encoder._spatial_latent = net.encoder.spatial_encoder          # the frozen ResNet once per step, for comparison only
    g = torch.Generator().manual_seed(3)
    t = median_time(lambda: training.test_time_step(net, opt, batches.source_view_batch(views, src, generator=g)), repeats, warmup=2)
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    del net, opt
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    return {"kind": "test_time_step", "views": nv, "train_precision": train_precision, "resnet": "hoisted" if hoisted else "every step",
            "ms_per_step": 1e3 * t, "peak_gib": peak}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--views", type=int, nargs="+", default=[1, 3, 5])
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--fp32-rays", type=int, default=16384)
    ap.add_argument("--skip-render", action="store_true")
    ap.add_argument("--skip-tto", action="store_true")
    ap.add_argument("--json", default=None, help="also write the results to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_views.py measures on a CUDA device; there is no CPU fallback")
    dev = torch.device("cuda:0")
    gpu = card()
    print(f"card: {gpu}")
    res = []
    if not a.skip_render:
        for W, H in ((640, 480), (320, 240)):
            for nv in a.views:
                for prec in ("tc", "fp32"):
                    res.append(bench_render(dev, nv, W, H, prec, a.fp32_rays, a.repeats))
                    print(json.dumps(res[-1]), flush=True)
    if not a.skip_tto:
        for nv in a.views:
            for tp in ("fp32", "tc"):
                for hoisted in (True, False):
                    res.append(bench_tto(dev, nv, tp, hoisted, a.repeats))
                    print(json.dumps(res[-1]), flush=True)
    print(f"\n{gpu}")
    for r in res:
        if r["kind"] == "render":
            print(f"render {r['size']:>7}  NV={r['views']}  {r['precision']:>4}: {r['rays_per_s'] / 1e3:9.1f} k rays/s ({r['rays']} rays)")
        else:
            print(f"test-time step  NV={r['views']}  {r['train_precision']:>4}  ResNet {r['resnet']:>10}: {r['ms_per_step']:7.1f} ms"
                  f"  (peak {r['peak_gib']:.1f} GiB)")
    if a.json:
        with open(a.json, "w") as f:
            json.dump({"card": gpu, "results": res}, f, indent=1)


if __name__ == "__main__":
    main()
