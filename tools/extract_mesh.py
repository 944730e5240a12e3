"""Mesh the foreground of the bench scene (bench.py: 640x480 sources, 3 views, 120x160 tri-planes, seed 0) and write a PLY.

    python tools/extract_mesh.py --resolution 256 --out scene.ply                 # iso = median sigma inside the unit sphere
    python tools/extract_mesh.py --resolution 256 --iso 5.0 --precision fp32 --out scene.ply
    python tools/extract_mesh.py --time --json mesh_times.json                  # stage times, rates and peak memory

The synthetic scene has no trained density, so without --iso the tool takes a quantile of the grid's sigma inside the sphere.
--time times the three stages separately with a device synchronise around each repeat, after a warm-up of every shape: the density grid
(lattice points per second, fp32 and tc), marching tetrahedra (count + emit) and normals + colours, with the peak device memory of each.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def bench_net(dev, precision):
    from neo360_b200 import NeRF_TP, synth
    sc = synth.make_scene((640, 480), 3, (120, 160), seed=0)
    net = NeRF_TP(num_coarse_samples=128, num_fine_samples=64, num_src_views=3, precision=precision).eval()
    net.load_state_dict(synth.make_mlp_params(0))
    net = net.to(dev)
    net.set_scene(*[sc[k].to(dev) for k in ("planes_xz", "planes_xy", "planes_yz", "latent", "src_poses", "src_focal", "src_c")],
                  sc["img_wh"], precisions=["fp32", "tc"])
    return net


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


def iso_of(sigma, iso, q):
    # torch.quantile takes at most 2^24 values: the quantile of the first 2^24 positive ones (lattice order)
    return float(iso) if iso is not None else float(torch.quantile(sigma[sigma > 0].float()[:1 << 24], q))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--resolution", type=int, default=256)
    ap.add_argument("--precision", choices=("fp32", "tc"), default="tc")
    ap.add_argument("--level", type=int, default=1)
    ap.add_argument("--iso", type=float, default=None)
    ap.add_argument("--iso-quantile", type=float, default=0.5, help="without --iso: this quantile of sigma inside the unit sphere")
    ap.add_argument("--out", default=None, help="PLY path")
    ap.add_argument("--time", action="store_true", help="time the stages at several resolutions instead of writing one mesh")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--json", default=None, help="--time: also write the results here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("extract_mesh needs a CUDA device")
    from neo360_b200 import mesh, output
    dev = torch.device("cuda:0")
    net = bench_net(dev, args.precision)

    if not args.time:
        sigma = net.density_grid(args.resolution, level=args.level)
        iso = iso_of(sigma, args.iso, args.iso_quantile)
        m = mesh.extract_mesh(net, None, args.resolution, iso=iso, level=args.level)
        print(f"R={args.resolution} iso={iso:.6g}: {m['verts'].shape[0]} vertices, {m['faces'].shape[0]} faces")
        if args.out:
            print("wrote", output.write_ply(args.out, m))
        return

    res = {"device": torch.cuda.get_device_name(dev), "repeats": args.repeats, "grid": [], "mesh": []}
    try:
        import subprocess
        res["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                                            capture_output=True, text=True).stdout.strip()
    except OSError:
        res["power_limit"] = None
    for prec, Rs in (("fp32", (128, 256)), ("tc", (256, 512))):
        for R in Rs:
            sig, ts, peak = timed(lambda: net.density_grid(R, level=args.level, precision=prec), args.repeats)
            row = {"precision": prec, "R": R, "s": min(ts), "s_all": ts, "points_per_s": R ** 3 / min(ts), "peak_bytes": peak}
            res["grid"].append(row)
            print(json.dumps(row), flush=True)
    for R in (256, 512):
        sig = net.density_grid(R, level=args.level, precision="tc")
        iso = iso_of(sig, args.iso, args.iso_quantile)
        (v, f), ts_mt, peak_mt = timed(lambda: mesh.marching_tetrahedra(sig, iso), args.repeats)
        n, ts_n, _ = timed(lambda: mesh.grid_normals(sig, v), args.repeats)
        _, ts_c, peak_c = timed(lambda: mesh.vertex_colors(net, v, n, args.level, "tc"), args.repeats)
        row = {"R": R, "iso": iso, "V": v.shape[0], "F": f.shape[0], "mt_ms": 1e3 * min(ts_mt), "mt_ms_all": [1e3 * t for t in ts_mt],
               "normals_ms": 1e3 * min(ts_n), "colors_tc_ms": 1e3 * min(ts_c), "mt_peak_bytes": peak_mt, "colors_peak_bytes": peak_c}
        res["mesh"].append(row)
        print(json.dumps(row), flush=True)
        del sig, v, f, n
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
