"""GridEncoder training throughput on one GPU at the NeO-360 training shape: NV = 3 source views of 640 x 480 (latent 240 x 320),
the 64^3 grid, a fixed random loss on the three output planes.  Variants, alternated in the same run:
  * cuda_fp32 / cuda_tf32 / cuda_autocast: the CUDA form (`dense_train`: hand-written lookup and softmax pillar sums forward and backward,
    framework GEMMs) with fp32 GEMMs, TF32 GEMMs, and under torch.autocast(bfloat16);
  * tc: the tensor-core form (`dense_train_tc`, `GridEncoder(train_precision="tc")`: every dense layer a bf16 product of csrc/gemm_tc.cu);
  * torch_fp32 / torch_tf32: the framework form (`dense_torch`).

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
    # variant -> (dense-part method, TF32 GEMMs, autocast)
    variants = {"cuda_fp32": (enc.dense_train, False, False), "cuda_tf32": (enc.dense_train, True, False),
                "cuda_autocast": (enc.dense_train, False, True), "tc": (enc.dense_train_tc, False, False),
                "torch_fp32": (enc.dense_torch, False, False), "torch_tf32": (enc.dense_torch, True, False)}

    def dense_step(v):
        form, _, ac = variants[v]
        lat = latent0.clone().requires_grad_(True)
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=ac):
            planes = form(lat, poses, focal, c, W, H)
        sum((p.float() * w).sum() for p, w in zip(planes, w_dense)).backward()

    def encoder_step(v):
        form, _, ac = variants[v]
        enc.dense_train = form                              # forward() routes the dense part through this instance attribute
        enc.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=ac):
            out = enc(imgs, poses, focal, c)
        sum((o.float() * w).sum() for o, w in zip(out, w_out)).backward()
        del enc.dense_train

    res = {}
    r = {v: {"dense_ms": [], "encoder_ms": [], "peak_gb": 0.0} for v in variants}
    for _ in range(2):                                      # alternate the variants twice, keep the better time of each
        for v in variants:
            torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = variants[v][1]
            r[v]["dense_ms"].append(events(lambda: dense_step(v), args.steps, args.warmup))
            enc.zero_grad(set_to_none=True)
            torch.cuda.empty_cache()
            torch.cuda.reset_peak_memory_stats(dev)
            r[v]["encoder_ms"].append(events(lambda: encoder_step(v), args.steps, args.warmup))
            r[v]["peak_gb"] = max(r[v]["peak_gb"], torch.cuda.max_memory_allocated(dev) / 1e9)
            enc.zero_grad(set_to_none=True)
            torch.cuda.empty_cache()
    for v in variants:
        d, e = min(r[v]["dense_ms"]), min(r[v]["encoder_ms"])
        res[v] = {"dense_fwd_bwd_ms": round(d, 2), "encoder_fwd_bwd_ms": round(e, 2), "peak_mem_gb": round(r[v]["peak_gb"], 2),
                  "dense_whole_step_tflops": round(STEP_FLOP / (d * 1e-3) / 1e12, 1),
                  "dense_ms_runs": [round(x, 2) for x in r[v]["dense_ms"]], "encoder_ms_runs": [round(x, 2) for x in r[v]["encoder_ms"]]}
    for base in ("cuda_fp32", "cuda_tf32", "cuda_autocast"):
        res[f"tc_speedup_dense_vs_{base}"] = round(min(r[base]["dense_ms"]) / min(r["tc"]["dense_ms"]), 2)
    for prec in ("fp32", "tf32"):
        res[f"{prec}_speedup_dense"] = round(min(r[f"torch_{prec}"]["dense_ms"]) / min(r[f"cuda_{prec}"]["dense_ms"]), 2)
    print(json.dumps({"metric": "GridEncoder forward + backward, NV = 3, 640x480, 64^3 grid", "card": name, "power_limit_w": power,
                      "dense_step_flop": STEP_FLOP, "steps": args.steps, "warmup": args.warmup, **res}))


if __name__ == "__main__":
    main()
