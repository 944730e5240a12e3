"""Test-time optimisation of NeO-360 on the source views of a new scene (the reference's --is_optimize), on a synthetic scene.

    python tools/optimize_source_views.py --views 5 --steps 100
    python tools/optimize_source_views.py --views 1 --steps 50 --train-precision tc --lr 5e-4

A model with its GridEncoder is fine-tuned on its own NV source images: each step draws one source view and 500 of its pixels
(`batches.source_view_batch`, as the reference's dataset draws them), and takes a plain Adam step (`training.test_time_optimizer`:
ResNet-34 frozen and, with it, every BatchNorm in eval mode; no schedule, no clip).  The frozen ResNet runs once for the whole run.
The source images here are smooth random images and the weights are untrained, so the numbers only show the loop working: the MSE of a
fixed set of pixels of one source view is printed before and after.  Pass --lr 5e-4 to see it move within a few dozen steps; 5e-6, the
default, is the reference's rate for a model resumed from a checkpoint.
"""
import argparse
import os
import random
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def make_setup(dev, nv, img_wh=(640, 480), n_coarse=128, n_fine=256, train_precision="fp32", lr=None, seed=0):
    """(net, optimiser, source views as TargetViews, src dict) of a synthetic scene with NV smooth source images of size img_wh."""
    from neo360_b200 import NeRF_TP, batches, synth, training
    from neo360_b200.encoder import GridEncoder
    W, H = img_wh
    torch.manual_seed(seed)
    net = NeRF_TP(num_coarse_samples=n_coarse, num_fine_samples=n_fine, num_src_views=nv, precision="fp32",
                  train_precision=train_precision, encoder=GridEncoder(train_precision=train_precision))
    sd = net.state_dict()
    sd.update(synth.make_mlp_params(seed))
    net.load_state_dict(sd)
    net = net.to(dev).train()
    sc = synth.make_scene((W, H), nv, (4, 4), seed)           # cameras only: the encoder makes the feature maps
    g = torch.Generator().manual_seed(seed + 5)
    imgs = torch.nn.functional.interpolate(torch.rand(nv, 3, H // 8, W // 8, generator=g), size=(H, W), mode="bilinear",
                                           align_corners=False).clamp(0, 1).to(dev)
    views = batches.TargetViews(sc["src_poses"].to(dev), imgs.permute(0, 2, 3, 1), float(sc["src_focal"][0]))
    src = {k: sc[k].to(dev) for k in ("src_poses", "src_focal", "src_c")}
    src["src_imgs"] = imgs * 2 - 1                              # normalised, as the dataset hands the source images to the encoder
    opt = training.test_time_optimizer(net, **({} if lr is None else {"lr": lr}))
    return net, opt, views, src


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--views", type=int, default=5, choices=(1, 3, 5))
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--lr", type=float, default=None, help="default: training.TEST_TIME_LR (5e-6)")
    ap.add_argument("--train-precision", default="fp32", choices=("fp32", "tc"))
    ap.add_argument("--width", type=int, default=640)
    ap.add_argument("--height", type=int, default=480)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from neo360_b200 import batches, training
    dev = torch.device("cuda:0")
    net, opt, views, src = make_setup(dev, a.views, (a.width, a.height), train_precision=a.train_precision, lr=a.lr, seed=a.seed)
    random.seed(a.seed)
    torch.manual_seed(a.seed)
    probe = batches.source_view_batch(views, src, view=0, ray_batch_size=4096)

    def mse():
        with torch.no_grad():
            return float(((net(probe, False, False, None, None, out_depth=True)[1][0] - probe["target"]) ** 2).mean())

    print(f"{a.views} source views, {a.width}x{a.height}, train_precision={a.train_precision}, lr={opt.param_groups[0]['lr']:g}")
    print(f"view-0 MSE before: {mse():.6f}")
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for s in range(a.steps):
        loss = training.test_time_step(net, opt, batches.source_view_batch(views, src))
        if s % max(1, a.steps // 10) == 0 or s == a.steps - 1:
            print(f"step {s:4d}  loss {float(loss):.6f}")
    torch.cuda.synchronize()
    print(f"{a.steps} steps in {time.perf_counter() - t0:.2f} s")
    print(f"view-0 MSE after:  {mse():.6f}")


if __name__ == "__main__":
    main()
