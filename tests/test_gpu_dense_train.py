"""GPU: vanilla NeRF and Mip-NeRF 360 training with `train_precision="tc"` (csrc/dense_train.cu and gemm_tc.cu through
training._MLPTrainTC).

* each product form (forward with each epilogue, dgrad with and without the rank-1 addend, wgrad with the bias sums) within PRODUCT_BOUND
  of the float64 model at identical rounding points (oracle/dense_train_model.py), at the layer shapes of the three MLPs and at row
  counts that leave a partial 128-row tile;
* `_MLPTrainTC` forward within FWD_BOUND and every gradient within BWD_BOUND of the model (WIDE_ bounds for the 8 x 1024 Mip-NeRF 360
  NeRFMLP), for all three MLP kinds; two backward calls bit-identical;
* whole steps (vanilla configs[0]-shaped: 1024 rays, 64 + 64 samples; Mip-NeRF 360: 2048 rays, 64 / 64 / 32): every parameter gradient
  within STEP_BOUND of the "fp32" path's (each density bias together with its weight);
* convergence: teacher / student, 200 Adam steps per model, the final "tc" loss within 8 % of fp32's (the a-priori 10 %, tightened from
  the measured 0.8 % and 5.2 %);
* determinism: three Adam steps twice under torch.use_deterministic_algorithms(True), in a subprocess, bit-identical for both models;
* inference of a module trained with "tc" equals that of an "fp32" module loaded with the same state dict, bit for bit;
* errors: bad arguments are refused before any launch; train_precision="bogus" raises ValueError.
"""
import json
import os
import subprocess
import sys

import pytest
import torch

from oracle import dense_train_model as dtm

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def cuda():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from neo360_b200 import build
    build.build()
    return torch.device("cuda:0")


def lib():
    from neo360_b200 import _lib as L
    return L.load()


def bf16(x):
    return x.to(torch.bfloat16).contiguous()


def rand(*shape, seed, scale=1.0, dev):
    return (scale * torch.randn(*shape, generator=torch.Generator().manual_seed(seed))).to(dev)


# (M rows, N, K): the table's layer shapes at row counts that leave a partial 128-row tile
SHAPES = [(66560 + 37, 256, 64), (4133, 256, 256), (4133, 256, 320), (4133, 128, 256), (131072 + 5, 256, 512), (6001, 1024, 1024),
          (6001, 1024, 1536), (6001, 256, 1024)]


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_forward_product_against_model(cuda, M, N, K):
    s = torch.cuda.current_stream().cuda_stream
    A, W, b = bf16(torch.relu(rand(M, K, seed=1, dev=cuda))), bf16(rand(N, K, seed=2, scale=K ** -0.5, dev=cuda)), rand(N, seed=3, dev=cuda)
    ref = A.double() @ W.double().T + b.double()
    for epi in (0, 1, 2):
        C = torch.empty(M, N, device=cuda, dtype=torch.float32 if epi == 2 else torch.bfloat16)
        rc = lib().neo_tc_gemm_bf16(A.data_ptr(), K, W.data_ptr(), K, None if epi == 2 else b.data_ptr(), C.data_ptr(), N, M, N, K, epi, s)
        assert rc == 0
        want = ref - (b.double() if epi == 2 else 0)
        want = dtm.bf(torch.relu(want)) if epi == 0 else (dtm.bf(want) if epi == 1 else want)
        err = dtm.rel_err(C.double(), want)
        print("fwd", M, N, K, epi, err)
        assert err < dtm.PRODUCT_BOUND, (epi, err)


@pytest.mark.parametrize("M,N,K", [(4133, 256, 256), (6001, 1024, 1024), (6001, 1024, 256), (4133, 256, 128)])
def test_dgrad_against_model(cuda, M, N, K):
    """dX (M, N) = (dY (M, K) . W (K, N) + g w^T) [X > 0], W given as W^T (N, K)."""
    s = torch.cuda.current_stream().cuda_stream
    dY, Wt = bf16(rand(M, K, seed=4, scale=1e-3, dev=cuda)), bf16(rand(N, K, seed=5, scale=K ** -0.5, dev=cuda))
    X = bf16(torch.relu(rand(M, N + 64, seed=6, dev=cuda)))
    g, w = rand(M, seed=7, scale=1e-3, dev=cuda), rand(N, seed=8, dev=cuda)
    for addend in (False, True):
        for mask in (False, True):
            dX = torch.empty(M, N, device=cuda, dtype=torch.bfloat16)
            rc = lib().neo_tc_dgrad_bf16(dY.data_ptr(), K, Wt.data_ptr(), K, X.data_ptr() if mask else None, N + 64,
                                         g.data_ptr() if addend else None, w.data_ptr() if addend else None, dX.data_ptr(), N, M, N, K, s)
            assert rc == 0
            want = dY.double() @ Wt.double().T
            if addend:
                want = want + g.double()[:, None] * w.double()[None, :]
            if mask:
                want = want * (X[:, :N].double() > 0)
            err = dtm.rel_err(dX.double(), dtm.bf(want))
            print("dgrad", M, N, K, addend, mask, err)
            assert err < dtm.PRODUCT_BOUND, (addend, mask, err)


@pytest.mark.parametrize("M,N,K,kv", [(66560 + 37, 256, 64, 63), (4133, 256, 320, 319), (131072 + 5, 256, 512, 504), (6001, 1024, 1024, 1024),
                                      (6001, 1024, 1536, 1528), (4133, 128, 256, 256), (6001, 64, 1024, 1024)])
def test_wgrad_against_model(cuda, M, N, K, kv):
    s = torch.cuda.current_stream().cuda_stream
    dY, X = bf16(rand(M, N, seed=9, scale=1e-3, dev=cuda)), bf16(torch.relu(rand(M, K, seed=10, dev=cuda)))
    need = lib().neo_tc_wgrad_bf16_workspace_bytes(M, N, K)
    assert 0 < need <= (32 << 20) + 64 * N * 4 + 256
    ws = torch.empty(need, dtype=torch.uint8, device=cuda)
    dW, db = torch.empty(N, kv, device=cuda), torch.empty(N, device=cuda)
    assert lib().neo_tc_wgrad_bf16(dY.data_ptr(), N, X.data_ptr(), K, M, N, K, dW.data_ptr(), kv, db.data_ptr(), ws.data_ptr(), need, s) == 0
    e_w = dtm.rel_err(dW.double(), (dY.double().T @ X.double())[:, :kv])
    e_b = dtm.rel_err(db.double(), dY.double().sum(0))
    print("wgrad", M, N, K, e_w, e_b)
    assert e_w < dtm.PRODUCT_BOUND and e_b < dtm.PRODUCT_BOUND


def mlp_case(kind, n, N, seed, dev):
    from neo360_b200 import mip, vanilla
    torch.manual_seed(seed)
    m, F = (vanilla.NeRFMLP(), 63) if kind == "vanilla" else ((mip.PropMLP(), 504) if kind == "prop" else (mip.NeRFMLP(), 504))
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for p in m.parameters():
            p.add_(0.01 * torch.randn(p.shape, generator=g))
    feats = torch.randn(n * N, F, generator=g).clamp(-1, 1)
    denc = torch.randn(n, 27, generator=g)
    return m.to(dev), feats.to(dev), denc.to(dev)


def run_tc(m, feats, gs, gy):
    from neo360_b200 import training
    m.zero_grad(set_to_none=True)
    layers = m.pts_linears if hasattr(m, "pts_linears") else m.pts_linear
    params = [t for lin in layers for t in (lin.weight, lin.bias)] + [m.density_layer.weight, m.density_layer.bias]
    if hasattr(m, "rgb_layer"):
        v = m.views_linear[0]
        wvb = v.weight[:, :256].detach().clone().requires_grad_(True)
        params += [m.bottleneck_layer.weight, m.bottleneck_layer.bias, wvb]
        sig, yb = training._MLPTrainTC.apply(len(layers), feats, *params)
        (sig * gs).sum().add((yb * gy).sum()).backward()
    else:
        sig, yb = training._MLPTrainTC.apply(len(layers), feats, *params), None
        (sig * gs).sum().backward()
    G = {f"w{i}": l.weight.grad for i, l in enumerate(layers)}
    G.update({f"b{i}": l.bias.grad for i, l in enumerate(layers)})
    G.update(wsig=m.density_layer.weight.grad, bsig=m.density_layer.bias.grad)
    if yb is not None:
        G.update(wb=m.bottleneck_layer.weight.grad, bb=m.bottleneck_layer.bias.grad, wvb=wvb.grad)
    return sig.detach(), None if yb is None else yb.detach(), {k: v.clone() for k, v in G.items()}


@pytest.mark.parametrize("kind,n,N", [("vanilla", 1037, 65), ("vanilla", 1037, 129), ("prop", 2048, 64), ("mip", 2048, 32), ("mip", 517, 32)])
def test_mlp_against_model(cuda, kind, n, N):
    m, feats, _ = mlp_case(kind, n, N, 3, cuda)
    M = n * N
    gs = rand(M, 1, seed=11, scale=1e-3, dev=cuda)
    gy = rand(M, 128, seed=12, scale=1e-3, dev=cuda)
    sig, yb, G = run_tc(m, feats, gs, gy)
    P = dtm.params_of(m)                                   # the float64 model runs on the GPU too
    s_ref, y_ref, S = dtm.forward(feats.double(), P)
    G_ref = dtm.backward(gs.double(), gy.double() if y_ref is not None else None, S, P)
    errs = {"sigma": dtm.rel_err(sig, s_ref)}
    if y_ref is not None:
        errs["y_beta"] = dtm.rel_err(yb, y_ref)
    errs.update({k: dtm.rel_err(G[k], G_ref[k]) for k in G_ref})
    print("dense_train errors", kind, n, N, json.dumps({k: round(v, 6) for k, v in errs.items()}))
    fb, bb = (dtm.WIDE_FWD_BOUND, dtm.WIDE_BWD_BOUND) if kind == "mip" else (dtm.FWD_BOUND, dtm.BWD_BOUND)
    assert errs["sigma"] < fb and errs.get("y_beta", 0) < fb, errs
    for k in G_ref:
        assert errs[k] < bb, (k, errs)


def test_backward_bit_identical(cuda):
    for kind in ("vanilla", "prop"):
        m, feats, _ = mlp_case(kind, 1031, 64, 4, cuda)
        gs, gy = rand(1031 * 64, 1, seed=13, scale=1e-3, dev=cuda), rand(1031 * 64, 128, seed=14, scale=1e-3, dev=cuda)
        a, b = run_tc(m, feats, gs, gy), run_tc(m, feats, gs, gy)
        assert torch.equal(a[0], b[0])
        for k in a[2]:
            assert torch.equal(a[2][k], b[2][k]), (kind, k)


def test_bad_arguments(cuda):
    L = lib()
    s = torch.cuda.current_stream().cuda_stream
    buf = torch.zeros(1 << 22, dtype=torch.uint8, device=cuda)
    p = buf.data_ptr()
    assert L.neo_tc_gemm_bf16(p, 64, p, 64, None, p, 64, 8, 64, 48, 0, s) == -1            # K % 64
    assert L.neo_tc_gemm_bf16(p, 64, p, 64, None, p, 64, 8, 64, 64, 3, s) == -1            # unknown epilogue
    assert L.neo_tc_gemm_bf16(p + 2, 64, p, 64, None, p, 64, 8, 64, 64, 0, s) == -1        # misaligned A
    assert b"gemm_bf16" in L.neo_last_error()
    assert L.neo_tc_dgrad_bf16(p, 64, p, 64, None, 0, p, None, p, 64, 8, 64, 64, s) == -1  # g_sig without w_sig
    assert L.neo_tc_dgrad_bf16(p, 64, p, 64, p, 32, None, None, p, 64, 8, 64, 64, s) == -1  # ldx < N
    assert b"dgrad_bf16" in L.neo_last_error()
    assert L.neo_tc_wgrad_bf16_workspace_bytes(100, 96, 64) == 0                            # N % 64
    assert L.neo_tc_wgrad_bf16_workspace_bytes(0, 64, 64) == 0
    assert L.neo_tc_wgrad_bf16_workspace_bytes(100, 4096, 4096) == 0                        # partials past 32 MB
    need = L.neo_tc_wgrad_bf16_workspace_bytes(100, 64, 64)
    assert need > 0
    assert L.neo_tc_wgrad_bf16(p, 64, p, 64, 100, 64, 64, p, 64, None, p, need - 1, s) == -3
    assert L.neo_tc_wgrad_bf16(p, 64, p, 64, 100, 64, 64, p, 65, None, p, need, s) == -1   # k_valid > K
    assert L.neo_tc_wgrad_bf16(p, 64, p, 64, 100, 64, 64, None, 64, None, p, need, s) == -1
    assert b"wgrad_bf16" in L.neo_last_error()
    assert L.neo_tc_pack_bf16(p, 4, 8, 8, p, 16, 8, 0, s) == -1                              # ld_out < cols_out
    assert L.neo_tc_pack_bf16(p, 4, 8, 8, p, 16, 4, 1, s) == -1                              # transpose: cols_out > cols_in
    assert L.neo_tc_relu_rank1_bf16(p, p, None, 64, 8, 64, p, 64, s) == -1
    assert L.neo_tc_rowdot_bf16(p, 256, 256, p, p, 2, 8, p, s) == -1
    assert b"rowdot_bf16" in L.neo_last_error()
    torch.cuda.synchronize()


def test_bogus_train_precision():
    from neo360_b200.mip import MipNeRF360
    from neo360_b200.vanilla import NeRF
    with pytest.raises(ValueError, match="train_precision"):
        NeRF(train_precision="bogus")
    with pytest.raises(ValueError, match="train_precision"):
        MipNeRF360(train_precision="bogus")


# ---- whole models ----

def vanilla_net(dev, prec, seed=0):
    from neo360_b200 import synth
    from neo360_b200.vanilla import NeRF
    net = NeRF(num_coarse_samples=64, num_fine_samples=64, train_precision=prec)
    net.load_state_dict(synth.make_vanilla_params(seed))
    return net.to(dev).train()


def mip_net(dev, prec, seed=0):
    from neo360_b200 import synth
    from neo360_b200.mip import MipNeRF360
    net = MipNeRF360(num_prop_samples=64, num_nerf_samples=32, train_precision=prec)
    net.load_state_dict(synth.make_mip_params(seed))
    return net.to(dev).train()


def vanilla_batch(dev, n, seed=0):
    from tools.bench_vanilla_train import crop_batch
    rays, target = crop_batch(dev)
    idx = torch.randint(0, rays["rays_o"].shape[0], (n,), generator=torch.Generator().manual_seed(seed)).to(dev)
    return {k: v[idx] for k, v in rays.items()}, target[idx]


def mip_batch(dev, n, seed=0):
    from tools.bench_mip_train import ray_pool
    rays, target = ray_pool(dev)
    idx = torch.randint(0, rays["rays_o"].shape[0], (n,), generator=torch.Generator().manual_seed(seed)).to(dev)
    return {k: v[idx] for k, v in rays.items()}, target[idx]


def vanilla_loss(net, batch, target, randomized=True):
    ret = net(batch, randomized, True, 2.0, 6.0)
    return ((ret[0][0] - target) ** 2).mean() + ((ret[1][0] - target) ** 2).mean()


def mip_loss(net, batch, target, randomized=True):
    from neo360_b200.mip import training_loss
    ren, hist = net(batch, 0.5, randomized, True, 0.2, 100.0)
    return training_loss(ren, hist, target)


MODELS = {"vanilla": (vanilla_net, vanilla_batch, vanilla_loss, 1024), "mip": (mip_net, mip_batch, mip_loss, 2048)}


@pytest.mark.parametrize("model", ["vanilla", "mip"])
def test_whole_step_against_fp32(cuda, model):
    make, batch_of, loss_of, n = MODELS[model]
    batch, target = batch_of(cuda, n)
    grads = {}
    for prec in ("fp32", "tc"):
        net = make(cuda, prec)
        torch.manual_seed(0)
        loss_of(net, batch, target).backward()
        grads[prec] = {k: p.grad.clone() for k, p in net.named_parameters() if p.grad is not None}
        del net
    # a density layer's bias gradient is one scalar, the sum of a signed per-sample gradient that nearly cancels: its relative error says
    # nothing, so it is held to the bound together with its layer's weight gradient
    for g in grads.values():
        for k in [k for k in g if k.endswith("density_layer.bias")]:
            w = k.replace(".bias", ".weight")
            g[w] = torch.cat([g[w].reshape(-1), g.pop(k).reshape(-1)])
    errs = {k: dtm.rel_err(grads["tc"][k], grads["fp32"][k]) for k in grads["fp32"]}
    print("whole step", model, json.dumps({k: round(v, 5) for k, v in sorted(errs.items(), key=lambda kv: -kv[1])[:10]}))
    assert set(grads["tc"]) == set(grads["fp32"])
    for k, v in errs.items():
        assert v < dtm.STEP_BOUND, (k, v)


@pytest.mark.parametrize("model", ["vanilla", "mip"])
def test_convergence(cuda, model):
    """Teacher (params seed 1) renders the targets without jitter; the student starts from seed 0; 200 Adam steps."""
    make, batch_of, loss_of, n = MODELS[model]
    batch, _ = batch_of(cuda, 512)
    with torch.no_grad():
        teacher = make(cuda, "fp32", seed=1).eval()
        target = teacher(batch, False, True, 2.0, 6.0)[1][0] if model == "vanilla" else teacher(batch, 0.5, False, False, 0.2, 100.0)[0][-1]["rgb"]
    curves = {}
    for prec in ("fp32", "tc"):
        net = make(cuda, prec)
        opt = torch.optim.Adam(net.parameters(), lr=5e-4)
        losses = []
        for _ in range(200):
            loss = loss_of(net, batch, target, randomized=False)
            opt.zero_grad(set_to_none=True)
            loss.backward()
            opt.step()
            losses.append(float(loss.detach()))
        curves[prec] = losses
    print("convergence", model, json.dumps({k: [round(v[i], 6) for i in (0, 50, 100, 150, 199)] for k, v in curves.items()}))
    f32, tc = curves["fp32"], curves["tc"]
    assert f32[-1] < f32[0] and tc[-1] < tc[0]
    # a priori 10 %; measured on an H100: vanilla 0.000258 against 0.000256 (0.8 %), Mip-NeRF 360 0.003102 against 0.003273 (5.2 %)
    assert abs(tc[-1] - f32[-1]) <= 0.08 * f32[-1]


DET_SCRIPT = r"""
import json, sys, torch
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[1] + "/tests")
torch.use_deterministic_algorithms(True)
from test_gpu_dense_train import MODELS
dev = torch.device("cuda:0")
res = {}
for model in ("vanilla", "mip"):
    make, batch_of, loss_of, n = MODELS[model]
    batch, target = batch_of(dev, 512)
    out = []
    for run in range(2):
        net = make(dev, "tc")
        opt = torch.optim.Adam(net.parameters(), lr=5e-4)
        torch.manual_seed(0)
        rec = []
        for s in range(3):
            loss = loss_of(net, batch, target)
            opt.zero_grad(set_to_none=True)
            loss.backward()
            opt.step()
            rec.append(loss.item())
        out.append((rec, torch.cat([p.detach().reshape(-1) for p in net.parameters()]).cpu()))
    res[model] = out[0][0] == out[1][0] and torch.equal(out[0][1], out[1][1])
print(json.dumps(res))
"""


def test_deterministic_steps(cuda):
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    res = subprocess.run([sys.executable, "-c", DET_SCRIPT, ROOT], capture_output=True, text=True, env=env, timeout=900)
    assert res.returncode == 0, res.stderr[-3000:]
    r = json.loads(res.stdout.strip().splitlines()[-1])
    assert r == {"vanilla": True, "mip": True}, r


@pytest.mark.parametrize("model", ["vanilla", "mip"])
def test_inference_unchanged_by_train_precision(cuda, model):
    make, batch_of, loss_of, n = MODELS[model]
    batch, target = batch_of(cuda, 256)

    def infer(net):
        with torch.no_grad():
            net.eval()
            if model == "vanilla":
                out = [t for lvl in net(batch, False, True, 2.0, 6.0) for t in lvl]
            else:
                ren, hist = net(batch, 0.5, False, False, 0.2, 100.0)
                out = [r["rgb"] for r in ren] + [h["density"] for h in hist]
            net.train()
        return out

    tc = make(cuda, "tc")
    for step in range(2):
        ref = make(cuda, "fp32")
        ref.load_state_dict(tc.state_dict())
        a, b = infer(tc), infer(ref)
        assert all(torch.equal(x, y) for x, y in zip(a, b)), (model, step)
        if step == 0:
            opt = torch.optim.Adam(tc.parameters(), lr=5e-4)
            loss_of(tc, batch, target).backward()
            opt.step()
