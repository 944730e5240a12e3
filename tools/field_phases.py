"""Where the tensor-core field kernel spends its cycles: phase clocks of one bench.py frame.

Builds a copy of the library with -DNEO_FIELD_PHASES (clock64() marks in field_tc_kernel, see csrc/field_tc.cu) into a temporary
directory, loads it through NEO360_B200_LIB, renders the headline frame of bench.py (same scene, rays, img_wh block order and chunk)
once to warm up and once measured, and prints for each field launch the cycles per tile (64 points, all views) of every phase: the
consumer warpgroups' phases (blends and MMAs, and their waits for geometry) summed over the two consumers, and the producer's
phases (points, encodings, tap tables, and its waits for a free slot) summed over its two halves.  Whichever side waits less bounds
the tile.  It also prints the texel traffic the blends request: taps of non-zero weight per tile (each one 2 x 256 bytes, the P0
and P3 halves of a texel) over the cycles of the two blend phases, and how many of those taps a thread's two points share (the same
texel as the same tap of the other point, both weights non-zero: TapTable::share), which the blends fetch once for both points.
Usage on a GPU box:

  python tools/field_phases.py [--lib PATH] [--clock-mhz F]
      --lib: an instrumented library built beforehand, e.g. from another source tree
      --clock-mhz: SM clock the request rate is converted at (read it with nvidia-smi in the same run)
"""
import argparse
import ctypes as C
import os
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CONSUMER = ("waiting for geometry", "rows + encodings", "blend P0", "layers 0-2", "blend P3", "layer 3 + head", "direction term",
            "colour head + stores")
PRODUCER = ("setup", "encodings", "tap table", "waiting for a free slot")
PHASES = CONSUMER + PRODUCER                                         # column order of neo_field_phases_read (csrc/field_tc.cu)
LAUNCHES = ("fg coarse", "bg coarse", "fg fine", "bg fine")      # order of the field launches of one frame (render.cu)
MAX_LAUNCHES = 64


def build_instrumented(out_dir):
    from neo360_b200 import build as b
    path = os.path.join(out_dir, "libneo360_b200_phases.so")
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    cmd = [nvcc] + b.FLAGS + ["-DNEO_FIELD_PHASES", "-o", path] + [os.path.join(b.CSRC, s) for s in b.SOURCES]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + res.stdout + res.stderr)
    return path


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None, help="instrumented library to load instead of building one")
    ap.add_argument("--clock-mhz", type=float, default=1980.0, help="SM clock for the bytes/s figures")
    args = ap.parse_args()
    tmp = tempfile.TemporaryDirectory(prefix="neo360_phases_")
    os.environ["NEO360_B200_LIB"] = os.path.abspath(args.lib) if args.lib else build_instrumented(tmp.name)

    import torch
    import bench as Bm
    from neo360_b200 import NeRF_TP, _lib
    lib = _lib.load()
    if not hasattr(lib, "neo_field_phases_read"):
        raise RuntimeError(f"{os.environ['NEO360_B200_LIB']} was not built with -DNEO_FIELD_PHASES")
    lib.neo_field_phases_reset.restype = C.c_int
    lib.neo_field_phases_read.restype = C.c_int
    lib.neo_field_phases_read.argtypes = [C.POINTER(C.c_ulonglong), C.c_int]

    dev = torch.device("cuda:0")
    sc, P = Bm.build_scene_cpu()
    net = NeRF_TP(num_coarse_samples=Bm.N_COARSE, num_fine_samples=Bm.N_FINE, num_src_views=Bm.NV, precision="tc").eval()
    net.load_state_dict(P)
    net = net.to(dev)
    net.set_scene(*[sc[k].to(dev) for k in ("planes_xz", "planes_xy", "planes_yz", "latent", "src_poses", "src_focal", "src_c")],
                  sc["img_wh"])
    o, d = Bm.frame_rays_cpu(0)
    rays = {"rays_o": o.to(dev), "rays_d": d.to(dev), "viewdirs": d.to(dev)}
    wh = (Bm.IMG_W, Bm.IMG_H)
    with torch.no_grad():
        net.render_rays_test(rays, chunk=Bm.CHUNK, img_wh=wh)            # warm-up: module load, first-launch set-up
        torch.cuda.synchronize()
        if lib.neo_field_phases_reset() != 0:
            raise RuntimeError("neo_field_phases_reset failed")
        net.render_rays_test(rays, chunk=Bm.CHUNK, img_wh=wh)
        torch.cuda.synchronize()
    net.check()
    cols = len(PHASES) + 3                                               # phases, tiles, non-zero-weight taps, shared taps
    buf = (C.c_ulonglong * (MAX_LAUNCHES * cols))()
    n = lib.neo_field_phases_read(buf, MAX_LAUNCHES)
    if n < 0:
        raise RuntimeError("neo_field_phases_read failed")
    name = torch.cuda.get_device_name(0)
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    print(f"{name}; library {os.environ['NEO360_B200_LIB']}; {n} field launches; cycles per tile (64 points x {Bm.NV} views) per phase")
    rows = []
    for side, names, lo in (("consumers", CONSUMER, 0), ("producer", PRODUCER, len(CONSUMER))):
        print(f"{side}:")
        print(f"{'launch':<12}{'tiles':>9}" + "".join(f"{p:>24}" for p in names) + f"{'total':>12}")
        for li in range(n):
            row = buf[li * cols:(li + 1) * cols]
            tiles = max(row[-3], 1)
            per = [c / tiles for c in row[lo:lo + len(names)]]
            if lo == 0:
                rows.append((tiles, [c / tiles for c in row[:-3]], row[-2] / tiles, row[-1] / tiles))
            print(f"{LAUNCHES[li % 4]:<12}{row[-3]:>9}" + "".join(f"{x:>16.0f} ({x / max(sum(per), 1):4.0%})" for x in per)
                  + f"{sum(per):>12.0f}")
    # request rate of the blends: a warpgroup's texel bytes per tile over its blend cycles per tile; the GPU figure assumes both
    # warpgroups of every SM blend at once (an upper bound), the launch figure spreads the bytes over the whole tile
    print(f"texel requests ({n_sm} SMs, 2 consumer warpgroups each, SM clock {args.clock_mhz:.0f} MHz):")
    # a shared tap is fetched once for the thread's two points: the fetches saved are shared / taps, and the bytes below are fetched
    print(f"{'launch':<12}{'taps/tile':>10}{'shared/tile':>12}{'fetches saved':>14}{'KB/tile':>9}{'B/cycle in blends':>19}"
          f"{'GPU TB/s in blends':>20}{'GPU TB/s over tile':>20}")
    for li, (tiles, per, taps, shared) in enumerate(rows):
        by = (taps - shared) * 512
        blend = per[PHASES.index("blend P0")] + per[PHASES.index("blend P3")]
        scale = 2 * n_sm * args.clock_mhz * 1e6 / 1e12
        tile = sum(per[:len(CONSUMER)])
        print(f"{LAUNCHES[li % 4]:<12}{taps:>10.0f}{shared:>12.0f}{shared / max(taps, 1):>14.1%}{by / 1024:>9.0f}{by / blend:>19.1f}{by / blend * scale:>20.2f}{by / tile * scale:>20.2f}")


if __name__ == "__main__":
    main()
