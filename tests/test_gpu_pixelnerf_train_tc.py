"""GPU: PixelNeRF training with `train_precision="tc"` (the PixelNeRF form of csrc/field_train.cu through training._PixelTrunkTC).

* trunk: hbar within FWD_BOUND of the float64 model (oracle/pixelnerf_train_tc_model.py), d_p0 and every weight / bias
  gradient within BWD_BOUND of its adjoint, for NV 1, 3, 5 (and 8 once) and point counts that leave a partial 64-row tile; two
  backward calls bit-identical;
* bad arguments to the three entry points are refused before any launch;
* a whole 1024-ray, 64 + 64-sample, NV = 3 step with the real ResNet-34 trunk: every MLP parameter's gradient, the latent's and every
  encoder parameter's within STEP_BOUND of the "fp32" path's;
* convergence: teacher / student, 200 Adam steps, the final "tc" loss within 5 % of the fp32 run's (tightened from an a-priori 10 %; two
  runs on an H100 measured 0.03 % and 2.9 %: the lookup's atomic backward makes each run's last steps differ);
* determinism: three Adam steps twice under torch.use_deterministic_algorithms(True), in a subprocess, bit-identical;
* inference is unchanged: a "tc"-trained model and an "fp32" model loaded with its state dict render the same frames, bit for bit;
* an unknown train_precision raises.
"""
import copy
import json
import os
import subprocess
import sys

import pytest
import torch

from oracle import pixelnerf_train_tc_model as ptm

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = torch.device("cuda:0")
NEAR, FAR = 0.02, 3.0


@pytest.fixture(scope="module", autouse=True)
def built():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from neo360_b200 import build
    build.build()


def trunk_case(nv, M, seed):
    from neo360_b200.pixelnerf import NeRFMLP
    g = torch.Generator().manual_seed(seed)
    torch.manual_seed(seed)
    mlp = NeRFMLP()
    cam = torch.randn(nv, M, 3, generator=g)
    p0 = 0.3 * torch.randn(nv * M, 128, generator=g)
    return mlp.to(DEV), cam.to(DEV), p0.to(DEV)


def run_tc(mlp, cam, p0, g_hbar):
    from neo360_b200 import training
    p = mlp.pts_linears
    leaves = [t.detach().clone().requires_grad_(True) for t in (p[0].weight[:, :63], p[0].bias, p[1].weight, p[1].bias, p[2].weight,
                                                              p[2].bias, p[3].weight, p[3].bias)]
    p0l = p0.clone().requires_grad_(True)
    hbar = training._PixelTrunkTC.apply(cam, p0l, *leaves)
    hbar.backward(g_hbar)
    keys = ("w0e", "b0", "w1", "b1", "w2", "b2", "w3", "b3")
    return hbar.detach(), p0l.grad, {k: t.grad for k, t in zip(keys, leaves)}


CASES = [(1, 7 * 65), (1, 5 * 129), (3, 7 * 65), (3, 5 * 129), (5, 7 * 65), (5, 5 * 129), (8, 5 * 129)]


@pytest.mark.parametrize("nv,M", CASES)
def test_trunk_against_model(nv, M):
    mlp, cam, p0 = trunk_case(nv, M, 20 + nv)
    g = 1e-4 * torch.randn(M, 128, generator=torch.Generator().manual_seed(7)).to(DEV)
    hbar, d_p0, G = run_tc(mlp, cam, p0, g)
    W = ptm.weights_of(mlp.cpu())
    h_ref, S = ptm.forward(cam.cpu().double(), p0.cpu().double(), W)
    d_ref, G_ref = ptm.backward(g.cpu().double(), S, W)
    assert set(G) == set(G_ref)
    errs = {"hbar": ptm.rel_err(hbar.cpu(), h_ref), "d_p0": ptm.rel_err(d_p0.cpu(), d_ref)}
    errs.update({k: ptm.rel_err(G[k].cpu(), G_ref[k]) for k in G})
    print("pixelnerf train errors", nv, M, json.dumps({k: round(v, 6) for k, v in errs.items()}))
    assert errs["hbar"] < ptm.FWD_BOUND, errs
    for k, v in errs.items():
        assert v < ptm.BWD_BOUND, (k, errs)


def test_backward_bit_identical():
    mlp, cam, p0 = trunk_case(3, 5 * 129, 3)
    g = 1e-4 * torch.randn(5 * 129, 128, generator=torch.Generator().manual_seed(8)).to(DEV)
    a = run_tc(mlp, cam, p0, g)
    b = run_tc(mlp, cam, p0, g)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    for k in a[2]:
        assert torch.equal(a[2][k], b[2][k]), k


def test_bad_arguments():
    from neo360_b200 import _lib as L
    lib = L.load()
    ws = lib.neo_pixelnerf_train_workspace_bytes
    assert ws(0, 10, 0) == 0 and ws(9, 10, 0) == 0 and ws(3, 0, 0) == 0 and ws(3, 10, 2) == 0
    assert ws(8, (1 << 22) + 1, 0) == 0                                   # more than 2^25 rows
    nv, M = 2, 100
    need, sc = ws(nv, M, 0), ws(nv, M, 1)
    assert need > 0 and sc > 0
    buf = torch.zeros(need, dtype=torch.uint8, device=DEV)
    sbuf = torch.zeros(sc, dtype=torch.uint8, device=DEV)
    x = torch.zeros(nv * M * 128 + 4, device=DEV)
    w = torch.zeros(128 * 128, device=DEV)
    s = torch.cuda.current_stream().cuda_stream
    fargs = lambda nv_, M_, p0, saved, n: (x.data_ptr(), p0, nv_, M_, *[w.data_ptr()] * 8, x.data_ptr(), saved, n, s)
    xp, wp_, bp = x.data_ptr(), w.data_ptr(), buf.data_ptr()
    assert lib.neo_pixelnerf_train_fwd(*fargs(nv, M, xp, bp, need - 1)) == -3
    assert lib.neo_pixelnerf_train_fwd(*fargs(nv, M, xp, None, need)) == -1
    assert lib.neo_pixelnerf_train_fwd(*fargs(nv, M, None, bp, need)) == -1
    assert lib.neo_pixelnerf_train_fwd(*fargs(0, M, xp, bp, need)) == -1
    assert lib.neo_pixelnerf_train_fwd(*fargs(9, M, xp, bp, need)) == -1
    assert lib.neo_pixelnerf_train_fwd(*fargs(nv, 0, xp, bp, need)) == -1
    assert lib.neo_pixelnerf_train_fwd(*fargs(8, (1 << 22) + 1, xp, bp, need)) == -1
    assert lib.neo_pixelnerf_train_fwd(*fargs(nv, M, xp + 4, bp, need)) == -1      # p0 not 16-byte aligned
    bargs = lambda d_p0, scr, n: (xp, nv, M, wp_, wp_, wp_, bp, need, d_p0, *[wp_] * 8, scr, n, s)
    assert lib.neo_pixelnerf_train_bwd(*bargs(xp, sbuf.data_ptr(), sc - 1)) == -3
    assert lib.neo_pixelnerf_train_bwd(*bargs(xp, None, sc)) == -1
    assert lib.neo_pixelnerf_train_bwd(*bargs(None, sbuf.data_ptr(), sc)) == -1
    assert lib.neo_pixelnerf_train_bwd(*bargs(xp + 4, sbuf.data_ptr(), sc)) == -1  # d_p0 not 16-byte aligned
    assert b"neo_pixelnerf_train_bwd" in lib.neo_last_error()
    torch.cuda.synchronize()


def make_rays(W, H, B, seed, pose=2):
    from neo360_b200 import synth
    from oracle import neo360_oracle as orc
    ro, vd, rd, _ = orc.rays_from_pose(orc.ray_directions(H, W, 0.8 * W), synth.target_pose(pose, 100)[:3, :4])
    sel = torch.randperm(H * W, generator=torch.Generator().manual_seed(seed))[:B]
    return {"rays_o": ro[sel], "rays_d": rd[sel], "viewdirs": vd[sel]}


def make_net(prec, nc, nf, seed, nv=3):
    from neo360_b200 import PixelNeRF, synth
    torch.manual_seed(seed)
    net = PixelNeRF(num_coarse_samples=nc, num_fine_samples=nf, num_src_views=nv, train_precision=prec)
    net.load_state_dict({**net.state_dict(), **synth.make_pixelnerf_params(seed)})
    return net.to(DEV).train()


def make_batch(W, H, B, nc, nf, seed, nv=3):
    from neo360_b200 import synth
    sc = synth.make_scene((W, H), nv, (8, 8), seed)
    b = {k: v.to(DEV) for k, v in make_rays(W, H, B, seed).items()}
    g = torch.Generator().manual_seed(seed)
    b.update(src_imgs=torch.rand(nv, 3, H, W, generator=g).to(DEV), src_poses=sc["src_poses"].to(DEV), src_focal=sc["src_focal"].to(DEV),
             src_c=sc["src_c"].to(DEV))
    b["_uniforms"] = [torch.rand(B, nc + 1, generator=g).to(DEV), torch.rand(B, nf, generator=g).to(DEV)]
    return b, torch.rand(B, 3, generator=g).to(DEV), sc


def loss_of(ret, t):
    return ((ret[0][0] - t) ** 2).mean() + ((ret[1][0] - t) ** 2).mean()


def test_whole_step_against_fp32():
    """1024 rays, 64 + 64 samples, NV = 3, the real ResNet-34 trunk on 160x120 source images; TF32 off on both paths.  The fine level
    resamples from the coarse weights, and at this scene the inverse CDF turns the coarse level's small differences into different fine
    samples (the fine MLP's gradients then differ by up to 0.77 between the two paths, and by 0.13 between the fp32 path with and without
    TF32 matmuls, measured on an H100); so that the comparison
    measures the arithmetic of the two paths, the "tc" step reuses the fp32 step's fine sample distances."""
    tf32 = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        b, target, _ = make_batch(160, 120, 1024, 64, 64, 5)
        grads, t1 = {}, [None]
        for prec in ("fp32", "tc"):
            net = make_net(prec, 64, 64, 5)
            enc_forward, keep = net.encoder.forward, {}

            def forward(x):
                keep["latent"] = enc_forward(x)
                keep["latent"].retain_grad()
                return keep["latent"]

            net.encoder.forward = forward
            sample = net._sample

            def pinned(lvl, *a):
                if lvl == 0:
                    return sample(lvl, *a)
                if prec == "fp32":
                    keep["t1"] = t1[0] = sample(lvl, *a)
                return t1[0]

            net._sample = pinned
            loss_of(net(b, True, False, NEAR, FAR), target).backward()
            grads[prec] = {n: p.grad.clone() for n, p in net.named_parameters() if p.grad is not None}
            grads[prec]["latent"] = keep["latent"].grad.clone()
            del net, keep
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32
    assert set(grads["tc"]) == set(grads["fp32"])
    assert any(k.startswith("encoder.") for k in grads["fp32"]) and "fine_mlp.pts_linears.3.weight" in grads["fp32"]
    errs = {k: ptm.rel_err(grads["tc"][k], grads["fp32"][k]) for k in grads["fp32"]}
    print("pixelnerf whole step", json.dumps({k: round(v, 5) for k, v in sorted(errs.items(), key=lambda kv: -kv[1])[:12]}))
    for k, v in errs.items():
        assert v < ptm.STEP_BOUND, (k, v)


def test_convergence():
    """Teacher (make_pixelnerf_params(1)) renders the targets from a fixed latent; the student starts from seed 0; 200 Adam steps over
    the MLPs, 1024 rays, 32 + 16 samples."""
    from neo360_b200 import synth
    W, H, nv, B, nc, nf = 64, 48, 3, 1024, 32, 16
    b, _, sc = make_batch(W, H, B, nc, nf, 9)
    b.pop("_uniforms")
    latent = sc["latent"].to(DEV)
    teacher = make_net("fp32", nc, nf, 1).eval()
    teacher.encoder.forward = lambda x: latent
    with torch.no_grad():
        target = teacher(b, False, False, NEAR, FAR)[1][0]
    curves = {}
    for prec in ("fp32", "tc"):
        net = make_net(prec, nc, nf, 0)
        net.encoder.forward = lambda x: latent
        params = list(net.coarse_mlp.parameters()) + list(net.fine_mlp.parameters())
        opt = torch.optim.Adam(params, lr=5e-4)
        losses = []
        for _ in range(200):
            loss = loss_of(net(b, False, False, NEAR, FAR), target)
            opt.zero_grad(set_to_none=True)
            loss.backward()
            opt.step()
            losses.append(float(loss.detach()))
        curves[prec] = losses
    print("pixelnerf convergence", json.dumps({k: [round(v[i], 6) for i in (0, 50, 100, 150, 199)] for k, v in curves.items()}))
    f32, tc = curves["fp32"], curves["tc"]
    assert f32[-1] < 0.3 * f32[0] and tc[-1] < 0.3 * tc[0]
    assert abs(tc[-1] - f32[-1]) <= 0.05 * f32[-1]         # measured on an H100: 0.006402 / 0.006589 against 0.006404 (0.03 % / 2.9 %)


DET_SCRIPT = r"""
import json, sys, torch
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[1] + "/tests")
torch.use_deterministic_algorithms(True)
from test_gpu_pixelnerf_train_tc import make_net, make_batch, loss_of, NEAR, FAR
out = []
for run in range(2):
    b, target, _ = make_batch(64, 48, 512, 32, 16, 4)
    net = make_net("tc", 32, 16, 2)
    opt = torch.optim.Adam(net.parameters(), lr=5e-4)
    rec = []
    for s in range(3):
        loss = loss_of(net(b, True, False, NEAR, FAR), target)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
        rec.append(loss.item())
    state = [t.detach().float().reshape(-1).cpu() for st in opt.state.values() for k, t in sorted(st.items()) if torch.is_tensor(t)]
    flat = torch.cat([p.detach().reshape(-1).cpu() for p in net.parameters()] + state)
    out.append((rec, flat))
same = out[0][0] == out[1][0] and torch.equal(out[0][1], out[1][1])
print(json.dumps({"same": same, "losses": out[0][0]}))
"""


def test_deterministic_steps():
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    res = subprocess.run([sys.executable, "-c", DET_SCRIPT, ROOT], capture_output=True, text=True, env=env, timeout=900)
    assert res.returncode == 0, res.stderr[-3000:]
    r = json.loads(res.stdout.strip().splitlines()[-1])
    assert r["same"], r


def test_inference_unchanged_by_training_precision():
    """Two Adam steps in "tc"; an "fp32" model loaded with the state dict renders bit-identical frames in precision fp32 and tc."""
    W, H, nv, nc, nf = 64, 48, 3, 32, 16
    b, target, _ = make_batch(W, H, 256, nc, nf, 6)
    a = make_net("tc", nc, nf, 6)
    opt = torch.optim.Adam(a.parameters(), lr=5e-4)
    for _ in range(2):
        loss = loss_of(a(b, True, False, NEAR, FAR), target)
        opt.zero_grad()
        loss.backward()
        opt.step()
    c = make_net("fp32", nc, nf, 7)
    c.load_state_dict(copy.deepcopy(a.state_dict()))
    a.eval(), c.eval()
    frame = {k: v.to(DEV) for k, v in make_rays(W, H, W * H, 0, pose=5).items()}
    frame.update({k: b[k] for k in ("src_imgs", "src_poses", "src_focal", "src_c")})
    for prec in ("fp32", "tc"):
        a.precision = c.precision = prec
        with torch.no_grad():
            ra, rc = a(frame, False, False, NEAR, FAR), c(frame, False, False, NEAR, FAR)
        for lvl in range(2):
            for i in range(3):
                assert torch.equal(ra[lvl][i], rc[lvl][i]), (prec, lvl, i)


def test_invalid_train_precision():
    from neo360_b200 import PixelNeRF
    with pytest.raises(ValueError, match="train_precision"):
        PixelNeRF(train_precision="bf16")
    b, _, _ = make_batch(64, 48, 64, 16, 8, 3)
    net = make_net("fp32", 16, 8, 3)
    net.train_precision = "fp16"
    with pytest.raises(ValueError, match="train_precision"):
        net(b, True, False, NEAR, FAR)
