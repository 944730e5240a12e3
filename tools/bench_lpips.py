"""LPIPS on one GPU, the CUDA head (neo_lpips_prepare + neo_lpips_head) against the framework form the reference runs (torch scaling and
`head_torch`), both on the same VGG-16 trunk (framework convolutions), alternated in one run.  Seeded weights in the real files' shapes;
timings do not depend on the weight values.

  * eval LPIPS per frame over 100 frames (`output.lpips_each`, one frame at a time as LitModel.lpips_each runs them) at 640 x 480 and
    1280 x 960, with cuDNN TF32 on (the default the reference runs under) and off;
  * the head alone on one frame pair's features, and the peak memory each head form adds on top of the features;
  * one NeO-360 fine-tuning step (900-ray patch, GridEncoder in the step with its spatial encoder frozen, Adam, clip 0.05) with and
    without the LPIPS term.
Times come from CUDA events after warm-up.  Prints one JSON line with the card name and power limit; writes nothing.

    python tools/bench_lpips.py [--frames 100] [--reps 20] [--steps 10]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from neo360_b200 import output
from neo360_b200.lpips import LPIPS, head, head_torch
from oracle import lpips_model as lm
from tools.bench_metrics import timed
from tools.bench_vanilla_train import card

SIZES = [(480, 640), (960, 1280)]
MEAN = torch.tensor(lm.MEAN).view(1, 3, 1, 1)
STD = torch.tensor(lm.STD).view(1, 3, 1, 1)


def framework_lpips(model, x, y):
    """piqa's LPIPS in framework ops on one (H, W, 3) pair: clamp, permute, (x - mean) / std, the trunk, head_torch."""
    def prep(t):
        t = torch.clip(t.permute(2, 0, 1).unsqueeze(0), 0, 1)
        return (t - MEAN.to(t.device)) / STD.to(t.device)
    return head_torch(model.trunk(prep(x)), model.trunk(prep(y)), [w for w in model.lin])


def framework_lpips_each(model, preds, gts):
    with torch.no_grad():
        return torch.stack([framework_lpips(model, p, g)[0] for p, g in zip(preds, gts)]).cpu()


def peak_extra(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def finetune_step_ms(dev, with_lpips, lp, steps, warmup):
    import bench as Bm
    from neo360_b200 import NeRF_TP, batches, synth, training
    from neo360_b200.encoder import GridEncoder
    torch.manual_seed(0)
    net = NeRF_TP(num_coarse_samples=Bm.N_COARSE, num_fine_samples=Bm.N_FINE, num_src_views=Bm.NV, precision="fp32", encoder=GridEncoder())
    sd = net.state_dict()
    sd.update(synth.make_mlp_params(0))
    net.load_state_dict(sd)
    net = net.to(dev).train()
    params = training.setup_finetune_lpips(net)
    opt = torch.optim.Adam(params, lr=5e-6)
    sc = synth.make_scene((Bm.IMG_W, Bm.IMG_H), Bm.NV, (120, 160), 0)
    src = {k: sc[k].to(dev) for k in ("src_poses", "src_focal", "src_c")}
    src["src_imgs"] = (torch.rand(Bm.NV, 3, Bm.IMG_H, Bm.IMG_W, generator=torch.Generator().manual_seed(77)) * 2 - 1).to(dev)
    g = torch.Generator().manual_seed(1234)
    tposes = torch.stack([synth.target_pose(5 * k, 100)[:3, :4] for k in range(batches.NUM_TARGET_VIEWS)]).to(dev)
    views = batches.TargetViews(tposes, torch.rand(batches.NUM_TARGET_VIEWS, Bm.IMG_H, Bm.IMG_W, 3, generator=g).to(dev), 0.8 * Bm.IMG_W)
    state = {"k": 0}

    def step():
        k = state["k"] = state["k"] + 1
        batch = batches.patch_batch(views, src, k % batches.NUM_TARGET_VIEWS)
        ret = net(batch, True, False, None, None, out_depth=False)
        loss = training.training_loss(ret, batch["target"], lpips_model=lp if with_lpips else None)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        torch.nn.utils.clip_grad_norm_(params, 0.05)
        opt.step()

    ms = timed(step, steps, warmup)
    del net, opt
    torch.cuda.empty_cache()
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=100)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_lpips needs a CUDA device"
    dev = torch.device("cuda:0")
    name, watts = card(dev)
    model = LPIPS()
    model.load_vgg16(lm.vgg16_state(0))
    model.load_lin(lm.lin_state(lm.lin_weights(0), "lpips"))
    model = model.to(dev)
    tf32_default = torch.backends.cudnn.allow_tf32
    res = {"card": name, "power_limit_w": watts, "cudnn_allow_tf32_default": tf32_default, "eval": [], "head": [], "finetune": {}}
    for H, W in SIZES:
        gen = torch.Generator(device=dev).manual_seed(H)
        x = torch.rand(args.frames, H, W, 3, device=dev, generator=gen)
        y = (0.8 * x + 0.3 * torch.rand(args.frames, H, W, 3, device=dev, generator=gen) - 0.05).contiguous()
        preds, gts = list(x), list(y)
        for tf32 in (True, False):
            torch.backends.cudnn.allow_tf32 = tf32
            t = {"cuda": 0.0, "framework": 0.0}
            for _ in range(2):      # alternate the forms
                t["cuda"] += timed(lambda: output.lpips_each(preds, gts, model), 1, 1) / 2
                t["framework"] += timed(lambda: framework_lpips_each(model, preds, gts), 1, 1) / 2
            a, b = output.lpips_each(preds, gts, model).double(), framework_lpips_each(model, preds, gts).double()
            res["eval"].append({"H": H, "W": W, "frames": args.frames, "cudnn_tf32": tf32,
                                "cuda_ms_per_frame": round(t["cuda"] / args.frames, 3),
                                "framework_ms_per_frame": round(t["framework"] / args.frames, 3),
                                "max_rel_diff": float(((a - b).abs() / b.abs()).max())})
        torch.backends.cudnn.allow_tf32 = tf32_default
        with torch.no_grad():
            from neo360_b200.lpips import prepare
            fx, fy = model.trunk(prepare(x[:1])), model.trunk(prepare(y[:1]))
        ws = [w.contiguous() for w in model.lin]
        feat_bytes = sum(f.numel() * 4 for f in fx + fy)
        hc = timed(lambda: head(fx, fy, ws), args.reps, args.warmup)
        ht = timed(lambda: head_torch(fx, fy, ws), args.reps, args.warmup)
        hc2 = timed(lambda: head(fx, fy, ws), args.reps, args.warmup)
        res["head"].append({"H": H, "W": W, "feature_bytes": feat_bytes, "cuda_ms": round(min(hc, hc2), 4), "framework_ms": round(ht, 4),
                            "cuda_read_gbps": round(2 * feat_bytes / (min(hc, hc2) * 1e-3) / 1e9, 1),
                            "cuda_peak_extra_bytes": peak_extra(lambda: head(fx, fy, ws)),
                            "framework_peak_extra_bytes": peak_extra(lambda: head_torch(fx, fy, ws))})
        del x, y, preds, gts, fx, fy
        torch.cuda.empty_cache()
    for tf32 in (True, False):
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = tf32
        a = finetune_step_ms(dev, True, model, args.steps, args.warmup)
        b = finetune_step_ms(dev, False, model, args.steps, args.warmup)
        res["finetune"]["tf32" if tf32 else "fp32"] = {"with_lpips_ms": round(a, 2), "without_lpips_ms": round(b, 2)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
