"""GPU: NeO-360 training with `train_precision="tc"` (csrc/field_train.cu through training._TrunkTC).

* forward: hbar within FWD_BOUND of the float64 model (oracle/field_train_model.py) for fg / bg, NV 1, 3, 5, N = 129 and 193 samples of
  a ray count that leaves a partial 64-row tile;
* backward: d_pm and every weight / bias gradient within BWD_BOUND of the model's adjoint; two calls bit-identical;
* a whole configs[3]-shaped step (4096 rays, 128 + 64 samples, frozen encoder): every MLP parameter's gradient and the feature maps'
  gradients within STEP_BOUND of the "fp32" path's;
* convergence: a teacher / student run, 200 Adam steps, the final "tc" loss within 2 % of the fp32 run's (the issue's a-priori 10 %, tightened from the measured 0.07 %);
* determinism: three Adam steps twice under torch.use_deterministic_algorithms(True), in a subprocess, bit-identical;
* errors: bad arguments are refused before any launch, and "tc" without the projected formulation raises.
"""
import json
import os
import subprocess
import sys

import pytest
import torch

from oracle import field_train_model as ftm

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def cuda():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from neo360_b200 import build
    build.build()
    return torch.device("cuda:0")


def trunk_case(ich, nv, M, seed, dev):
    from neo360_b200.renderer import NeRFPPMLP
    g = torch.Generator().manual_seed(seed)
    torch.manual_seed(seed)
    mlp = NeRFPPMLP(0, 10, 4, num_src_views=nv, input_ch=ich)
    cam = torch.randn(nv, M, ich, generator=g)
    lp = 0.3 * torch.randn(nv * M, 256, generator=g)
    wp = 0.3 * torch.randn(nv * M, 256, generator=g)
    return mlp.to(dev), cam.to(dev), lp.to(dev), wp.to(dev)


def run_tc(mlp, cam, lp, wp, g_hbar):
    from neo360_b200 import training
    ich = cam.shape[-1]
    E = 21 * ich
    p = mlp.pts_linears
    leaves = [t.detach().clone().requires_grad_(True) for t in (p[0].weight[:, :E], p[0].bias, p[1].weight, p[1].bias, p[2].weight,
                                                              p[2].bias, p[3].weight[:, :128 + E], p[3].bias)]
    lpl, wpl = lp.clone().requires_grad_(True), wp.clone().requires_grad_(True)
    hbar = training._TrunkTC.apply(cam, lpl, wpl, *leaves)
    hbar.backward(g_hbar)
    keys = ("w0e", "b0", "w1", "b1", "w2", "b2", "w3e", "b3")
    return hbar.detach(), lpl.grad, wpl.grad, {k: t.grad for k, t in zip(keys, leaves)}


CASES = [(3, 1, 7 * 129), (4, 1, 7 * 129), (3, 3, 7 * 129), (4, 3, 5 * 193), (3, 5, 5 * 193), (4, 5, 7 * 129)]


@pytest.mark.parametrize("ich,nv,M", CASES)
def test_trunk_against_model(cuda, ich, nv, M):
    mlp, cam, lp, wp = trunk_case(ich, nv, M, 10 + nv, cuda)
    g = 1e-4 * torch.randn(M, 128, generator=torch.Generator().manual_seed(7)).to(cuda)
    hbar, g_lp, g_wp, G = run_tc(mlp, cam, lp, wp, g)
    W = ftm.weights_of(mlp.cpu(), ich)
    h_ref, S = ftm.forward(cam.cpu().double(), lp.cpu().double(), wp.cpu().double(), W)
    d_ref, G_ref = ftm.backward(g.cpu().double(), S, W)
    errs = {"hbar": ftm.rel_err(hbar.cpu(), h_ref), "d_pm": ftm.rel_err(g_lp.cpu(), d_ref)}
    errs.update({k: ftm.rel_err(G[k].cpu(), G_ref[k]) for k in G})
    print("field_train errors", ich, nv, M, json.dumps({k: round(v, 6) for k, v in errs.items()}))
    assert torch.equal(g_lp, g_wp)
    assert errs["hbar"] < ftm.FWD_BOUND, errs
    for k, v in errs.items():
        assert v < ftm.BWD_BOUND, (k, errs)


def test_backward_bit_identical(cuda):
    mlp, cam, lp, wp = trunk_case(4, 3, 5 * 193, 3, cuda)
    g = 1e-4 * torch.randn(5 * 193, 128, generator=torch.Generator().manual_seed(8)).to(cuda)
    a = run_tc(mlp, cam, lp, wp, g)
    b = run_tc(mlp, cam, lp, wp, g)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    for k in a[3]:
        assert torch.equal(a[3][k], b[3][k]), k


def test_bad_arguments(cuda):
    from neo360_b200 import _lib as L
    lib = L.load()
    assert lib.neo_field_train_workspace_bytes(0, 10, 3, 0) == 0
    assert lib.neo_field_train_workspace_bytes(9, 10, 3, 0) == 0
    assert lib.neo_field_train_workspace_bytes(3, 10, 5, 0) == 0
    assert lib.neo_field_train_workspace_bytes(3, 0, 3, 0) == 0
    nv, M, ich = 2, 100, 3
    need = lib.neo_field_train_workspace_bytes(nv, M, ich, 0)
    assert need > 0
    buf = torch.zeros(need, dtype=torch.uint8, device=cuda)
    x = torch.zeros(nv * M * 256, device=cuda)
    w = torch.zeros(128 * 256, device=cuda)
    s = torch.cuda.current_stream().cuda_stream
    args = lambda nv_, M_, ich_, ws, n: (x.data_ptr(), x.data_ptr(), x.data_ptr(), nv_, M_, ich_, *[w.data_ptr()] * 8, x.data_ptr(), ws, n, s)
    assert lib.neo_field_train_fwd(*args(nv, M, ich, buf.data_ptr(), need - 1)) == -3
    assert lib.neo_field_train_fwd(*args(nv, M, ich, None, need)) == -1
    assert lib.neo_field_train_fwd(*args(0, M, ich, buf.data_ptr(), need)) == -1
    assert lib.neo_field_train_fwd(*args(9, M, ich, buf.data_ptr(), need)) == -1
    assert lib.neo_field_train_fwd(*args(nv, M, 5, buf.data_ptr(), need)) == -1
    assert lib.neo_field_train_fwd(*args(nv, 0, ich, buf.data_ptr(), need)) == -1
    sc = lib.neo_field_train_workspace_bytes(nv, M, ich, 1)
    sbuf = torch.zeros(sc, dtype=torch.uint8, device=cuda)
    bargs = lambda scr, n: (x.data_ptr(), nv, M, ich, *[w.data_ptr()] * 3, buf.data_ptr(), need, x.data_ptr(), *[w.data_ptr()] * 8, scr, n, s)
    assert lib.neo_field_train_bwd(*bargs(sbuf.data_ptr(), sc - 1)) == -3
    assert lib.neo_field_train_bwd(*bargs(None, sc)) == -1
    torch.cuda.synchronize()


def make_net(dev, precision, n_coarse=128, n_fine=64, seed_params=0):
    from neo360_b200 import NeRF_TP, synth
    net = NeRF_TP(num_coarse_samples=n_coarse, num_fine_samples=n_fine, num_src_views=3, precision="fp32", train_precision=precision)
    sd = net.state_dict()
    sd.update(synth.make_mlp_params(seed_params))
    net.load_state_dict(sd)
    return net.to(dev).train()


def make_batch(dev, n_rays, seed=0):
    from neo360_b200 import batches, synth
    sc = synth.make_scene((640, 480), 3, (120, 160), seed=0)
    maps = {k: sc[k].to(dev).requires_grad_(True) for k in ("planes_xz", "planes_xy", "planes_yz", "latent")}
    g = torch.Generator().manual_seed(1234 + seed)
    tposes = torch.stack([synth.target_pose(5 * k, 100)[:3, :4] for k in range(batches.NUM_TARGET_VIEWS)]).to(dev)
    timgs = torch.rand(batches.NUM_TARGET_VIEWS, 480, 640, 3, generator=g).to(dev)
    views = batches.TargetViews(tposes, timgs, 0.8 * 640)
    src = {"src_poses": sc["src_poses"].to(dev), "src_focal": sc["src_focal"].to(dev), "src_c": sc["src_c"].to(dev),
           "src_imgs": torch.empty(3, 3, 480, 640, device="meta")}
    batch = batches.train_batch(views, src, pix_inds=batches.draw_pix_inds(views.T, views.H, views.W, n_rays, g))
    batch.update(maps)
    return batch, maps


def test_whole_step_against_fp32(cuda):
    from neo360_b200 import training
    batch, maps = make_batch(cuda, 4096)
    grads = {}
    for prec in ("fp32", "tc"):
        net = make_net(cuda, prec)
        torch.manual_seed(0)
        for t in maps.values():
            t.grad = None
        ret = net(batch, True, False, None, None, out_depth=False)
        training.training_loss(ret, batch["target"]).backward()
        grads[prec] = {n: p.grad.clone() for n, p in net.named_parameters() if p.grad is not None}
        grads[prec].update({k: t.grad.clone() for k, t in maps.items()})
        del net, ret
    errs = {k: ftm.rel_err(grads["tc"][k], grads["fp32"][k]) for k in grads["fp32"]}
    print("whole step", json.dumps({k: round(v, 5) for k, v in sorted(errs.items(), key=lambda kv: -kv[1])[:12]}))
    assert set(grads["tc"]) == set(grads["fp32"])
    for k, v in errs.items():
        assert v < ftm.STEP_BOUND, (k, v)


def test_out_depth_under_autograd(cuda):
    batch, _ = make_batch(cuda, 256)
    net = make_net(cuda, "tc", 32, 16)
    ret = net(batch, True, False, None, None, out_depth=True)
    ret[1][5].sum().backward()
    assert all(torch.isfinite(p.grad).all() for p in net.parameters() if p.grad is not None)


def test_tc_needs_projected(cuda):
    batch, _ = make_batch(cuda, 64)
    net = make_net(cuda, "tc", 16, 8)
    net.train_projected = False
    with pytest.raises(ValueError, match="projected"):
        net(batch, True, False, None, None)


def test_convergence(cuda):
    """Teacher (synth.make_mlp_params(1)) renders the targets; the student starts from seed 0; 200 Adam steps, frozen encoder."""
    from neo360_b200 import training
    batch, maps = make_batch(cuda, 1024)
    for t in maps.values():
        t.requires_grad_(False)
    teacher = make_net(cuda, "fp32", 32, 16, seed_params=1)
    target = teacher(batch, False, False, None, None)[1][0].detach()
    curves = {}
    for prec in ("fp32", "tc"):
        net = make_net(cuda, prec, 32, 16, seed_params=0)
        params = [p for m in net._mlps() for p in m.parameters()]
        opt = torch.optim.Adam(params, lr=5e-4)
        losses = []
        for step in range(200):
            ret = net(batch, False, False, None, None)
            loss = ((ret[1][0] - target) ** 2).mean() + ((ret[0][0] - target) ** 2).mean()
            opt.zero_grad(set_to_none=True)
            loss.backward()
            opt.step()
            losses.append(float(loss.detach()))
        curves[prec] = losses
    print("convergence", json.dumps({k: [round(v[i], 6) for i in (0, 50, 100, 150, 199)] for k, v in curves.items()}))
    f32, tc = curves["fp32"], curves["tc"]
    assert f32[-1] < 0.3 * f32[0] and tc[-1] < 0.3 * tc[0]
    assert abs(tc[-1] - f32[-1]) <= 0.02 * f32[-1]         # measured on an H100: 0.012336 against 0.012345 (0.07 %)


DET_SCRIPT = r"""
import json, sys, torch
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[1] + "/tests")
torch.use_deterministic_algorithms(True)
from test_gpu_field_train import make_net, make_batch
from neo360_b200 import training
dev = torch.device("cuda:0")
out = []
for run in range(2):
    batch, maps = make_batch(dev, 1024)
    net = make_net(dev, "tc", 64, 32)
    params = [p for m in net._mlps() for p in m.parameters()]
    opt = torch.optim.Adam(params, lr=5e-4)
    torch.manual_seed(0)
    rec = []
    for s in range(3):
        ret = net(batch, True, False, None, None)
        loss = training.training_loss(ret, batch["target"])
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
        rec.append(loss.item())
    flat = torch.cat([p.detach().reshape(-1) for p in params] + [t.grad.reshape(-1) for t in maps.values()])
    out.append((rec, flat.cpu()))
same = out[0][0] == out[1][0] and torch.equal(out[0][1], out[1][1])
print(json.dumps({"same": same, "losses": out[0][0]}))
"""


def test_deterministic_steps(cuda):
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    res = subprocess.run([sys.executable, "-c", DET_SCRIPT, ROOT], capture_output=True, text=True, env=env, timeout=900)
    assert res.returncode == 0, res.stderr[-3000:]
    r = json.loads(res.stdout.strip().splitlines()[-1])
    assert r["same"], r
