"""GridEncoder training throughput on one GPU at the NeO-360 training shape: NV = 3 source views of 640 x 480 (latent 240 x 320),
the 64^3 grid, a fixed random loss on the three output planes.  The CUDA form (`dense_train`: hand-written lookup and softmax pillar sums
forward and backward, framework GEMMs) and the framework form (`dense_torch`) alternate in the same run, in fp32 and with TF32 GEMMs.

Per form and precision it reports, from CUDA events after warm-up:
  * the dense part's forward + backward (latent -> three floor plans; the ResNet and the conv stacks excluded) and the whole
    `GridEncoder` forward + backward, in ms;
  * the peak `torch.cuda.max_memory_allocated` of the whole forward + backward;
  * a whole-step FLOP rate of the dense part: 3 x 2 x the MACs of its dense layers (forward and the two backward GEMMs), computed from
    the layer shapes below, over the dense part's time (a whole-step rate, not a kernel's share of peak);
and the card name and power limit read in the same run.  Prints one JSON line; writes nothing.

    python tools/bench_encoder_train.py [--steps 10] [--warmup 3]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from neo360_b200 import synth
from neo360_b200.encoder import GridEncoder
from tools.bench_vanilla_train import card

NV, W, H, G = 3, 640, 480, 64
ROWS = NV * G ** 3
# per grid row: depth_fc 518->512->512->512, three aggregators 513->512->1
MAC_PER_ROW = 518 * 512 + 512 * 512 + 512 * 512 + 3 * (513 * 512 + 512)
STEP_FLOP = 3 * 2 * MAC_PER_ROW * ROWS


def events(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_encoder_train needs a CUDA device")
    dev = torch.device("cuda:0")
    name, power = card(dev)
    torch.manual_seed(0)
    enc = GridEncoder().train().to(dev)
    sc = synth.make_scene((W, H), NV, (4, 4), 0)
    poses, focal, c = sc["src_poses"].to(dev), sc["src_focal"].to(dev), sc["src_c"].to(dev)
    gen = torch.Generator().manual_seed(1)
    imgs = (torch.rand(NV, 3, H, W, generator=gen) * 2 - 1).to(dev)
    w_dense = [torch.randn(NV, 512, G, G, generator=gen).to(dev) for _ in range(3)]
    w_out = [torch.randn(NV, 128, 120, 160, generator=gen).to(dev) for _ in range(3)]
    with torch.no_grad():
        latent0 = enc.spatial_encoder(imgs).detach()
    forms = {"cuda": enc.dense_train, "torch": enc.dense_torch}

    def dense_step(form):
        lat = latent0.clone().requires_grad_(True)
        planes = forms[form](lat, poses, focal, c, W, H)
        sum((p * w).sum() for p, w in zip(planes, w_dense)).backward()

    def encoder_step(form):
        enc.dense_train = forms[form]
        enc.zero_grad(set_to_none=True)
        out = enc(imgs, poses, focal, c)
        sum((o * w).sum() for o, w in zip(out, w_out)).backward()
        del enc.dense_train

    res = {}
    for prec in ("fp32", "tf32"):
        torch.backends.cuda.matmul.allow_tf32 = prec == "tf32"
        torch.backends.cudnn.allow_tf32 = prec == "tf32"
        r = {f: {"dense_ms": [], "encoder_ms": [], "peak_gb": 0.0} for f in forms}
        for _ in range(2):                                  # alternate the two forms twice, keep the better time of each
            for f in forms:
                r[f]["dense_ms"].append(events(lambda: dense_step(f), args.steps, args.warmup))
                enc.zero_grad(set_to_none=True)
                torch.cuda.empty_cache()
                torch.cuda.reset_peak_memory_stats(dev)
                r[f]["encoder_ms"].append(events(lambda: encoder_step(f), args.steps, args.warmup))
                r[f]["peak_gb"] = max(r[f]["peak_gb"], torch.cuda.max_memory_allocated(dev) / 1e9)
                enc.zero_grad(set_to_none=True)
                torch.cuda.empty_cache()
        for f in forms:
            d, e = min(r[f]["dense_ms"]), min(r[f]["encoder_ms"])
            res[f"{prec}_{f}"] = {"dense_fwd_bwd_ms": round(d, 2), "encoder_fwd_bwd_ms": round(e, 2), "peak_mem_gb": round(r[f]["peak_gb"], 2),
                                  "dense_whole_step_tflops": round(STEP_FLOP / (d * 1e-3) / 1e12, 1),
                                  "dense_ms_runs": [round(x, 2) for x in r[f]["dense_ms"]], "encoder_ms_runs": [round(x, 2) for x in r[f]["encoder_ms"]]}
        res[f"{prec}_speedup_dense"] = round(min(r["torch"]["dense_ms"]) / min(r["cuda"]["dense_ms"]), 2)
        res[f"{prec}_speedup_encoder"] = round(min(r["torch"]["encoder_ms"]) / min(r["cuda"]["encoder_ms"]), 2)
    print(json.dumps({"metric": "GridEncoder forward + backward, NV = 3, 640x480, 64^3 grid", "card": name, "power_limit_w": power,
                      "dense_step_flop": STEP_FLOP, "steps": args.steps, "warmup": args.warmup, **res}))


if __name__ == "__main__":
    main()
