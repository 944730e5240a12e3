"""Mesh one of the project's models with seeded synthetic weights and write a PLY, or time the meshing stages.

    python tools/extract_mesh.py --model neo360 --resolution 256 --out scene.ply      # iso = median sigma inside the unit sphere
    python tools/extract_mesh.py --model mip360 --half-extent 2 --resolution 256 --out mip.ply
    python tools/extract_mesh.py --model vanilla --iso 5.0 --precision fp32 --out vanilla.ply
    python tools/extract_mesh.py --time --json mesh_times.json                       # every model: stage times, rates and peak memory

Models (all seeded, no trained density): neo360 is the bench scene (640x480 sources, 3 views, 120x160 tri-planes, seed 0), vanilla and
mip360 the reference architectures with synth.make_*_params(0), pixelnerf the same 3 source views with the synthetic encoder output.
Without --iso the tool takes a quantile of the grid's sigma: inside the unit sphere for neo360 (its grid is 0 outside), over the whole
bbox for the other models.  --time times each stage separately with a device synchronise around each repeat, after a warm-up of every
shape: the density grid (lattice points per second) per model, precision and resolution, then marching tetrahedra (count + emit),
normals and vertex colours at R = 256 in "tc", with the peak device memory of each.  Grids whose fp32 run would take minutes are
reported as not measured.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

MODELS = ("neo360", "vanilla", "mip360", "pixelnerf")
# resolutions timed per model and precision; the missing ones are "not measured" (minutes per grid on the fp32 CUDA-core paths)
TIMED = {("neo360", "fp32"): (128, 256), ("neo360", "tc"): (128, 256, 512),
         ("vanilla", "fp32"): (128, 256, 512), ("vanilla", "tc"): (128, 256, 512),
         ("mip360", "fp32"): (128, 256), ("mip360", "tc"): (128, 256, 512),
         ("pixelnerf", "fp32"): (128, 256), ("pixelnerf", "tc"): (128, 256, 512)}


def make_model(kind, dev, precision):
    """(net, batch) with seeded synthetic weights; batch is the source-view part PixelNeRF needs (None for the others)."""
    from neo360_b200 import synth
    if kind == "neo360":
        from neo360_b200 import NeRF_TP
        sc = synth.make_scene((640, 480), 3, (120, 160), seed=0)
        net = NeRF_TP(num_coarse_samples=128, num_fine_samples=64, num_src_views=3, precision=precision).eval()
        net.load_state_dict(synth.make_mlp_params(0))
        net = net.to(dev)
        net.set_scene(*[sc[k].to(dev) for k in ("planes_xz", "planes_xy", "planes_yz", "latent", "src_poses", "src_focal", "src_c")],
                      sc["img_wh"], precisions=["fp32", "tc"])
        return net, None
    if kind == "vanilla":
        from neo360_b200.vanilla import NeRF
        net = NeRF().eval()
        net.precision = precision
        net.load_state_dict(synth.make_vanilla_params(0))
        return net.to(dev), None
    if kind == "mip360":
        from neo360_b200.mip import MipNeRF360
        net = MipNeRF360(precision=precision).eval()
        net.load_state_dict(synth.make_mip_params(0))
        return net.to(dev), None
    from neo360_b200 import PixelNeRF
    sc = synth.make_scene((640, 480), 3, (120, 160), seed=0)
    net = PixelNeRF(num_src_views=3)
    net.load_state_dict({**net.state_dict(), **synth.make_pixelnerf_params(0)})
    net = net.to(dev).eval()
    net.precision = precision
    latent = sc["latent"].to(dev)
    net.encoder.forward = lambda x: latent                     # the synthetic encoder output stands in for the ResNet
    batch = {"src_imgs": torch.zeros(3, 3, 480, 640, device=dev), "src_poses": sc["src_poses"].to(dev),
             "src_focal": sc["src_focal"].to(dev), "src_c": sc["src_c"].to(dev)}
    return net, batch


def timed(fn, repeats):
    """(result of the last call, [seconds per call], peak bytes allocated during the calls)."""
    fn()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out, ts = None, []
    for _ in range(repeats):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return out, ts, torch.cuda.max_memory_allocated() - base


def iso_of(kind, sigma, iso, q):
    if iso is not None:
        return float(iso)
    vals = sigma[sigma > 0] if kind == "neo360" else sigma.reshape(-1)
    # torch.quantile takes at most 2^24 values: the quantile of the first 2^24 (lattice order)
    return float(torch.quantile(vals.float()[:1 << 24], q))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", choices=MODELS, default="neo360")
    ap.add_argument("--resolution", type=int, default=256)
    ap.add_argument("--precision", choices=("fp32", "tc"), default="tc")
    ap.add_argument("--level", type=int, default=None, help="default: the model's last level")
    ap.add_argument("--half-extent", type=float, default=1.0, help="the grid spans [-h, h]^3")
    ap.add_argument("--iso", type=float, default=None)
    ap.add_argument("--iso-quantile", type=float, default=0.5, help="without --iso: this quantile of the grid's sigma")
    ap.add_argument("--out", default=None, help="PLY path")
    ap.add_argument("--time", action="store_true", help="time the stages of every --models at several resolutions instead of one mesh")
    ap.add_argument("--models", default=",".join(MODELS), help="--time: comma-separated models")
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--json", default=None, help="--time: also write the results here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("extract_mesh needs a CUDA device")
    from neo360_b200 import mesh, output
    dev = torch.device("cuda:0")
    h = args.half_extent
    bbox = ((-h, -h, -h), (h, h, h))

    if not args.time:
        net, batch = make_model(args.model, dev, args.precision)
        sigma = mesh.density_grid(net, args.resolution, bbox, args.level, batch=batch)
        iso = iso_of(args.model, sigma, args.iso, args.iso_quantile)
        m = mesh.extract_mesh(net, batch, args.resolution, iso=iso, bbox=bbox, level=args.level)
        print(f"{args.model} R={args.resolution} iso={iso:.6g}: {m['verts'].shape[0]} vertices, {m['faces'].shape[0]} faces")
        if args.out:
            print("wrote", output.write_ply(args.out, m))
        return

    res = {"device": torch.cuda.get_device_name(dev), "repeats": args.repeats, "grid": [], "mesh": []}
    try:
        res["power_limit,clocks.max.sm"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                                                          capture_output=True, text=True).stdout.strip()
    except OSError:
        res["power_limit,clocks.max.sm"] = None
    print(json.dumps({k: res[k] for k in ("device", "power_limit,clocks.max.sm")}), flush=True)
    for kind in args.models.split(","):
        bb = ((-2.0,) * 3, (2.0,) * 3) if kind == "mip360" else bbox
        for prec in ("fp32", "tc"):
            net, batch = make_model(kind, dev, prec)
            for R in (128, 256, 512):
                row = {"model": kind, "precision": prec, "R": R}
                if R not in TIMED[(kind, prec)]:
                    row["s"] = "not measured"
                else:
                    _, ts, peak = timed(lambda: mesh.density_grid(net, R, bb, args.level, batch=batch), args.repeats)
                    row.update(s=min(ts), s_all=ts, points_per_s=R ** 3 / min(ts), peak_bytes=peak)
                res["grid"].append(row)
                print(json.dumps(row), flush=True)
            if prec == "tc":
                R = 256
                sig = mesh.density_grid(net, R, bb, args.level, batch=batch)
                iso = iso_of(kind, sig, args.iso, args.iso_quantile)
                (v, f), ts_mt, peak_mt = timed(lambda: mesh.marching_tetrahedra(sig, iso, bb), args.repeats)
                n, ts_n, _ = timed(lambda: mesh.grid_normals(sig, v, bb), args.repeats)
                var = mesh.grid_var(mesh.make_grid(R, bb)) if kind == "mip360" else None
                _, ts_c, peak_c = timed(lambda: mesh.vertex_colors(net, v, n, args.level, "tc", batch, var), args.repeats)
                row = {"model": kind, "R": R, "iso": iso, "V": v.shape[0], "F": f.shape[0], "mt_ms": 1e3 * min(ts_mt),
                       "normals_ms": 1e3 * min(ts_n), "colors_tc_ms": 1e3 * min(ts_c), "mt_peak_bytes": peak_mt, "colors_peak_bytes": peak_c}
                res["mesh"].append(row)
                print(json.dumps(row), flush=True)
                del sig, v, f, n
            del net, batch
            torch.cuda.empty_cache()
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
