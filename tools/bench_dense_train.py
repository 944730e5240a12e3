"""Vanilla NeRF (--model vanilla: tools/bench_vanilla_train.py's workload, 1024 rays, 64 + 64 samples) or Mip-NeRF 360 (--model mip:
tools/bench_mip_train.py's, 2048 rays, 64 / 64 / 32 samples) training steps with the MLPs in four arithmetics, alternated in one process
over --rounds rounds: "fp32" (framework GEMMs), "tf32" (the same in TF32), "autocast" (the framework MLP under torch.autocast(bfloat16))
and "tc" (train_precision="tc": csrc/dense_train.cu).  Reports per variant ms per step (CUDA events around whole steps), the MLP forward
time (CUDA events around the MLP calls of the forward pass), peak device memory and the final loss, with the card name and power limit
read in the same run.  One JSON line to stdout.

--kernels instead times the three product forms at the Mip-NeRF 360 NeRFMLP shape (65 536 rows, 1024 x 1024) with CUDA events over many
launches, beside torch.matmul in bf16 at the same shapes, and reports kernel rates in TFLOP/s computed from the shapes."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.bench_vanilla_train import card  # noqa: E402


def kernels(dev, reps):
    from neo360_b200 import _lib as L
    lib = L.load()
    s = torch.cuda.current_stream().cuda_stream
    M, N, K = 65536, 1024, 1024
    g = torch.Generator(device=dev).manual_seed(0)
    X = torch.relu(torch.randn(M, K, device=dev, generator=g)).bfloat16()
    W = (torch.randn(N, K, device=dev, generator=g) * K ** -0.5).bfloat16()
    dY = (torch.randn(M, N, device=dev, generator=g) * 1e-3).bfloat16()
    b = torch.zeros(N, device=dev)
    C = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
    need = lib.neo_tc_wgrad_bf16_workspace_bytes(M, N, K)
    ws = torch.empty(need, dtype=torch.uint8, device=dev)
    dW, db = torch.empty(N, K, device=dev), torch.empty(N, device=dev)
    forms = {
        "fwd": lambda: L.check(lib.neo_tc_gemm_bf16(X.data_ptr(), K, W.data_ptr(), K, b.data_ptr(), C.data_ptr(), N, M, N, K, 0, s)),
        "dgrad": lambda: L.check(lib.neo_tc_dgrad_bf16(dY.data_ptr(), N, W.data_ptr(), K, X.data_ptr(), K, None, None, C.data_ptr(), N, M, K, N, s)),
        "wgrad": lambda: L.check(lib.neo_tc_wgrad_bf16(dY.data_ptr(), N, X.data_ptr(), K, M, N, K, dW.data_ptr(), K, db.data_ptr(), ws.data_ptr(),
                                                       need, s)),
        "torch_fwd": lambda: torch.matmul(X, W.t()),
        "torch_dgrad": lambda: torch.matmul(dY, W),
        "torch_wgrad": lambda: torch.matmul(dY.t(), X),
    }
    out = {}
    for name, fn in forms.items():
        for _ in range(5):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / reps
        out[name] = {"ms": ms, "tflops": 2.0 * M * N * K / (ms * 1e-3) / 1e12}
    return {"shape": {"rows": M, "N": N, "K": K}, "kernel_rates": out}


def steps(a, dev):
    from neo360_b200 import mip, synth, training, vanilla
    if a.model == "vanilla":
        from tools.bench_vanilla_train import BATCH, NC, NEAR, FAR, NF, crop_batch
        rays, target = crop_batch(dev)

        def make(prec):
            net = vanilla.NeRF(num_coarse_samples=NC, num_fine_samples=NF, train_precision=prec)
            net.load_state_dict(synth.make_vanilla_params(0))
            return net.to(dev).train()

        def loss_of(net, batch, tgt):
            ret = net(batch, True, True, NEAR, FAR)
            return ((ret[0][0] - tgt) ** 2).mean() + ((ret[1][0] - tgt) ** 2).mean()
        mods = [vanilla]
    else:
        from tools.bench_mip_train import BATCH, FAR, NEAR, NN, NP, ray_pool
        rays, target = ray_pool(dev)

        def make(prec):
            net = mip.MipNeRF360(num_prop_samples=NP, num_nerf_samples=NN, train_precision=prec)
            net.load_state_dict(synth.make_mip_params(0))
            return net.to(dev).train()

        def loss_of(net, batch, tgt):
            ren, hist = net(batch, 0.5, True, True, NEAR, FAR)
            return mip.training_loss(ren, hist, tgt)
        mods = [mip]

    events = []

    def timed(fn):
        def w(*args, **kw):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            r = fn(*args, **kw)
            e.record()
            events.append((s, e))
            return r
        return w
    for m in mods:
        m._mlp_train = timed(m._mlp_train)
        m.mlp_train_tc = timed(m.mlp_train_tc)

    gen = torch.Generator(device=dev).manual_seed(1)

    def step(variant, net, opt):
        torch.backends.cuda.matmul.allow_tf32 = variant == "tf32"
        idx = torch.randint(0, rays["rays_o"].shape[0], (BATCH,), device=dev, generator=gen)
        batch, tgt = {k: v[idx] for k, v in rays.items()}, target[idx]
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=variant == "autocast"):
            loss = loss_of(net, batch, tgt)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
        return loss

    variants = a.variants.split(",")
    res = {v: {"ms": [], "mlp_fwd_ms": [], "peak_gb": 0.0, "loss": None} for v in variants}
    for _ in range(a.rounds):
        for v in variants:
            torch.manual_seed(0)
            net = make("tc" if v == "tc" else "fp32")
            opt = torch.optim.Adam(net.parameters(), lr=5e-4)
            for _ in range(a.warmup):
                step(v, net, opt)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            events.clear()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(a.steps):
                loss = step(v, net, opt)
            e.record()
            torch.cuda.synchronize()
            res[v]["ms"].append(s.elapsed_time(e) / a.steps)
            res[v]["mlp_fwd_ms"].append(sum(x.elapsed_time(y) for x, y in events) / a.steps)
            res[v]["peak_gb"] = max(res[v]["peak_gb"], torch.cuda.max_memory_allocated() / 2 ** 30)
            res[v]["loss"] = float(loss.detach())
            del net, opt
            torch.cuda.empty_cache()
    torch.backends.cuda.matmul.allow_tf32 = False
    return {"model": a.model, "rays": BATCH, "steps": a.steps, "rounds": a.rounds, "variants": res}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", choices=["vanilla", "mip"], default="vanilla")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--variants", default="fp32,tf32,autocast,tc")
    ap.add_argument("--kernels", action="store_true")
    ap.add_argument("--reps", type=int, default=50)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_dense_train.py measures on a CUDA device; none is available")
    dev = torch.device("cuda:0")
    out = kernels(dev, a.reps) if a.kernels else steps(a, dev)
    name, watts = card(dev)
    out.update(gpu=name, power_limit_w=watts)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
