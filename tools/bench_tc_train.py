"""NeO-360 training step (BASELINE configs[3]: 4096 rays, 128 + 64 samples, 3 source views) with the MLPs in four arithmetics, alternated
in one process: "fp32" (framework GEMMs, fp32), "tf32" (the same with TF32 GEMMs), "autocast" (the framework MLP under
torch.autocast(bfloat16)) and "tc" (train_precision="tc": csrc/field_train.cu).  The encoder is frozen (its outputs are leaf tensors) or,
with --encoder, runs inside the step; there a fifth variant, "tc_enc", trains both the MLPs and the encoder's dense part on the tensor
cores (`GridEncoder(train_precision="tc")`, csrc/encoder.cu around the bf16 products of csrc/gemm_tc.cu).  Reports ms per step (CUDA events around whole steps, after a device synchronise), the share of it
spent in the MLP forward (CUDA events around the MLP calls of the forward pass), peak device memory, and the GPU it ran on.
Writes one JSON line to stdout and, with --out, to that file."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--rays", type=int, default=4096)
    ap.add_argument("--encoder", action="store_true")
    ap.add_argument("--variants", default=None, help="default: fp32,tf32,autocast,tc, and tc_enc with --encoder")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from neo360_b200 import NeRF_TP, batches, synth, training
    from neo360_b200.encoder import GridEncoder
    dev = torch.device("cuda:0")
    sc = synth.make_scene((640, 480), 3, (120, 160), seed=0)
    g = torch.Generator().manual_seed(1234)
    tposes = torch.stack([synth.target_pose(5 * k, 100)[:3, :4] for k in range(batches.NUM_TARGET_VIEWS)]).to(dev)
    views = batches.TargetViews(tposes, torch.rand(batches.NUM_TARGET_VIEWS, 480, 640, 3, generator=g).to(dev), 0.8 * 640)
    src_imgs = (torch.rand(3, 3, 480, 640, generator=g) * 2 - 1).to(dev)

    # CUDA events around every MLP call of the forward pass
    mlp_events = []
    orig = {"fp32": training._mlp_projected, "tc": training._mlp_projected_tc}

    def timed(fn):
        def w(*args, **kw):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            r = fn(*args, **kw)
            e.record()
            mlp_events.append((s, e))
            return r
        return w
    training._mlp_projected, training._mlp_projected_tc = timed(orig["fp32"]), timed(orig["tc"])

    def make(variant):
        torch.manual_seed(0)
        enc = GridEncoder(train_precision="tc" if variant == "tc_enc" else "fp32") if a.encoder else None
        net = NeRF_TP(num_coarse_samples=128, num_fine_samples=64, num_src_views=3, precision="fp32", encoder=enc,
                      train_precision="tc" if variant in ("tc", "tc_enc") else "fp32")
        sd = net.state_dict()
        sd.update(synth.make_mlp_params(0))
        net.load_state_dict(sd)
        net = net.to(dev).train()
        maps = {} if a.encoder else {k: sc[k].to(dev).requires_grad_(True) for k in ("planes_xz", "planes_xy", "planes_yz", "latent")}
        params = [p for p in net.parameters() if p.requires_grad] if a.encoder else [p for m in net._mlps() for p in m.parameters()]
        return net, maps, params, torch.optim.Adam(params, lr=5e-4)

    def step(variant, net, maps, params, opt):
        torch.backends.cuda.matmul.allow_tf32 = variant == "tf32"
        torch.backends.cudnn.allow_tf32 = variant == "tf32"
        src = {"src_poses": sc["src_poses"].to(dev), "src_focal": sc["src_focal"].to(dev), "src_c": sc["src_c"].to(dev), "src_imgs": src_imgs}
        batch = batches.train_batch(views, src, pix_inds=batches.draw_pix_inds(views.T, views.H, views.W, a.rays, g))
        batch.update(maps)
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=variant == "autocast"):
            ret = net(batch, True, False, None, None)
            loss = training.training_loss(ret, batch["target"])
        opt.zero_grad(set_to_none=True)
        for t in maps.values():
            t.grad = None
        loss.backward()
        training.allreduce_flat(params, 1, None)
        torch.nn.utils.clip_grad_norm_(params, 0.05)
        opt.step()
        return loss

    variants = (a.variants or "fp32,tf32,autocast,tc" + (",tc_enc" if a.encoder else "")).split(",")
    res = {v: {"ms": [], "mlp_fwd_ms": [], "peak_gb": 0.0, "loss": None} for v in variants}
    for rnd in range(a.rounds):
        for v in variants:
            state = make(v)
            for _ in range(a.warmup):
                step(v, *state)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            mlp_events.clear()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(a.steps):
                loss = step(v, *state)
            e.record()
            torch.cuda.synchronize()
            res[v]["ms"].append(s.elapsed_time(e) / a.steps)
            res[v]["mlp_fwd_ms"].append(sum(x.elapsed_time(y) for x, y in mlp_events) / a.steps)
            res[v]["peak_gb"] = max(res[v]["peak_gb"], torch.cuda.max_memory_allocated() / 2 ** 30)
            res[v]["loss"] = float(loss.detach())
            del state
            torch.cuda.empty_cache()
    import subprocess
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    out = {"gpu": smi.stdout.strip(), "encoder": "in the step" if a.encoder else "frozen", "rays": a.rays, "steps": a.steps,
           "rounds": a.rounds, "variants": res}
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
