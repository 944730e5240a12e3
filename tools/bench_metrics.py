"""Evaluation metrics on one GPU: `ssim_each` and `psnr_obj_each` (hand-written CUDA) against the fp32 framework forms the reference
runs (piqa's SSIM as torch conv2d per frame, `oracle.metrics_model.ssim_framework`; `get_obj_rgbs_from_segmap` + `psnr_each` as torch
ops per frame), alternated in one run.  Workloads: 100 frames at 640 x 480 and 100 frames at 1280 x 960 (BASELINE configs[4], the
turntable size); frames are seeded correlated noise, masks a seeded random quarter of the pixels.

Per workload it reports, from CUDA events after warm-up (each timed call ends with the values on the host, as the callers use them):
  * ms per call for each form, and their ratio;
  * each SSIM form's largest per-frame error against the float64 model on the same frames, in absolute terms, for the framework form
    with the framework's default conv2d settings (TF32 when cudnn allows it, the precision the reference gets on an H100) and with TF32
    off;
  * the object PSNR's largest difference between the two forms;
and the card name and power limit read in the same run.  Prints one JSON line; writes nothing.

    python tools/bench_metrics.py [--reps 5] [--warmup 2]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from neo360_b200 import output
from oracle import metrics_model as mm
from tools.bench_vanilla_train import card

WORKLOADS = [(100, 480, 640), (100, 960, 1280)]


def timed(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def framework_ssim_each(preds, gts):
    return torch.stack([mm.ssim_framework(p[None], g[None])[1][0] for p, g in zip(preds, gts)]).cpu()


def framework_psnr_obj_each(preds, gts, masks):
    out = []
    for p, g, m in zip(preds, gts, masks):
        mk = m.unsqueeze(-1).repeat(1, 1, 3)
        mse = torch.mean((torch.clip(p[mk], 0, 1) - torch.clip(g[mk], 0, 1)) ** 2)
        out.append(-10.0 * torch.log(mse) / np.log(10))
    return torch.stack(out).cpu()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_metrics needs a CUDA device"
    dev = torch.device("cuda:0")
    name, watts = card(dev)
    res = {"card": name, "power_limit_w": watts, "cudnn_allow_tf32_default": torch.backends.cudnn.allow_tf32, "workloads": []}
    for n, H, W in WORKLOADS:
        g = torch.Generator(device=dev).manual_seed(n + H)
        x = torch.rand(n, H, W, 3, device=dev, generator=g)
        y = (0.8 * x + 0.3 * torch.rand(n, H, W, 3, device=dev, generator=g) - 0.05).contiguous()
        masks = torch.rand(n, H, W, device=dev, generator=g) < 0.25
        preds, gts, ms = list(x), list(y), list(masks)
        t = {"cuda_ssim": 0.0, "framework_ssim": 0.0, "cuda_psnr_obj": 0.0, "framework_psnr_obj": 0.0}
        for _ in range(2):      # alternate the forms
            t["cuda_ssim"] += timed(lambda: output.ssim_each(preds, gts), args.reps, args.warmup) / 2
            t["framework_ssim"] += timed(lambda: framework_ssim_each(preds, gts), args.reps, args.warmup) / 2
            t["cuda_psnr_obj"] += timed(lambda: output.psnr_obj_each(preds, gts, ms), args.reps, args.warmup) / 2
            t["framework_psnr_obj"] += timed(lambda: framework_psnr_obj_each(preds, gts, ms), args.reps, args.warmup) / 2
        ref = torch.stack([mm.ssim_f64(x[i], y[i])[1] for i in range(n)]).cpu()
        cuda_vals = output.ssim_batch(x, y).cpu()
        fw_default = framework_ssim_each(preds, gts).double()
        tf32 = torch.backends.cudnn.allow_tf32
        torch.backends.cudnn.allow_tf32 = False
        fw_fp32 = framework_ssim_each(preds, gts).double()
        torch.backends.cudnn.allow_tf32 = tf32
        obj_c, obj_f = output.psnr_obj_each(preds, gts, ms).double(), framework_psnr_obj_each(preds, gts, ms).double()
        res["workloads"].append({
            "frames": n, "H": H, "W": W, **{f"{k}_ms": round(v, 3) for k, v in t.items()},
            "ssim_speedup": round(t["framework_ssim"] / t["cuda_ssim"], 2),
            "psnr_obj_speedup": round(t["framework_psnr_obj"] / t["cuda_psnr_obj"], 2),
            "ssim_err_cuda": float((cuda_vals - ref).abs().max()),
            "ssim_err_framework_default": float((fw_default - ref).abs().max()),
            "ssim_err_framework_fp32": float((fw_fp32 - ref).abs().max()),
            "psnr_obj_max_diff_db": float((obj_c - obj_f).abs().max()),
        })
        del x, y, masks, preds, gts, ms
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
