"""GPU: GridEncoder's tensor-core training form (`GridEncoder(train_precision="tc")`, `dense_train_tc`) against the float64 model of its
bf16 numerics (oracle/encoder_train_tc_model.py, pinned to autograd through `dense_torch` on the CPU by
tests/test_encoder_train_tc_model.py), against the fp32 `dense_train`, inside the NeO-360 training step, in training and under
torch.use_deterministic_algorithms.

Bounds: the model's constants (DESIGN.md section 2 lists the card, its power limit and the measured values).  Run with `-m gpu -s`: every
comparison prints its measured maximum.
"""
import json
import os
import subprocess
import sys

import pytest
import torch

from neo360_b200 import synth
from oracle import encoder_train_model as etm
from oracle import encoder_train_tc_model as tcm
from test_gpu_encoder_train import compare_grads, dense_params, geometry, release_memory, shift_invariant  # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu

G = 64
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def cuda():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from neo360_b200 import build
    build.build()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    return torch.device("cuda:0")


def lib():
    from neo360_b200 import _lib as L
    return L.load()


@pytest.mark.parametrize("nv,lat_hw", [(1, (11, 18)), (3, (240, 320))])
def test_lookup_rows_are_rounded_fp32_rows(cuda, nv, lat_hw):
    """The bf16 lookup rows are bf16 of the fp32 entry's rows bit for bit (zeros past column 518); the coordinate fill writes the
    cell's bf16 x, y, z into columns 512..514 and zeros after them, leaving columns 0..511 alone."""
    from neo360_b200 import _lib as L
    poses, focal, c, W, H = geometry(nv, lat_hw)
    lh, lw = lat_hw
    R = nv * G ** 3
    lat_cl = (torch.rand(nv, lh, lw, 512, generator=torch.Generator().manual_seed(nv)) * 4 - 1).to(cuda)
    pc = poses.float().contiguous().to(cuda)
    args = (nv, lh, lw, W, H, L.ptr(pc), float(focal[0]), float(c[0, 0]), float(c[0, 1]))
    X = torch.empty(R, 520, device=cuda)
    Xb = torch.full((R, 576), 7.0, dtype=torch.bfloat16, device=cuda)
    L.check(lib().neo_grid_encoder_features(L.ptr(lat_cl), *args, L.ptr(X), 520, None))
    L.check(lib().neo_grid_encoder_features_bf16(L.ptr(lat_cl), *args, Xb.data_ptr(), 576, None))
    assert torch.equal(Xb[:, :518], X[:, :518].bfloat16())
    assert bool((Xb[:, 518:] == 0).all())
    L.check(lib().neo_grid_encoder_coords_bf16(Xb.data_ptr(), nv, 576, None))
    assert torch.equal(Xb[:, :512], X[:, :512].bfloat16())
    assert torch.equal(Xb[:, 512:515], tcm.grid_coords(G, nv, device=cuda).bfloat16())
    assert bool((Xb[:, 515:] == 0).all())
    print(f"lookup rows nv={nv} latent {lh}x{lw}: bf16 rows bit-identical to bf16(fp32 rows)")


@pytest.mark.parametrize("nv", [1, 3])
def test_pool_bf16_matches_model(cuda, nv):
    """The bf16 pool reads lat from L (row stride 576): forward and backward within POOL_BOUND of the model at identical inputs,
    bit-identical to the fp32 entries on the same values, and two backward calls bit-identical."""
    from neo360_b200 import _lib as L
    R = nv * G ** 3
    gen = torch.Generator().manual_seed(20 + nv)
    Lb = torch.randn(R, 576, generator=gen).to(cuda).bfloat16()
    lat = Lb[:, :512].float().contiguous()
    logits = (torch.rand(3, R, generator=gen) * 8 - 4).to(cuda)
    out = [torch.empty(nv, 512, G, G, device=cuda) for _ in range(3)]
    ref = [torch.empty(nv, 512, G, G, device=cuda) for _ in range(3)]
    L.check(lib().neo_grid_encoder_pool_bf16(Lb.data_ptr(), 576, L.ptr(logits), nv, *[L.ptr(t) for t in out], None))
    L.check(lib().neo_grid_encoder_pool(L.ptr(lat), L.ptr(logits), nv, *[L.ptr(t) for t in ref], None))
    assert all(torch.equal(a, b) for a, b in zip(out, ref))
    ups = [torch.randn(nv, 512, G, G, generator=gen).to(cuda) for _ in range(3)]
    runs = []
    for _ in range(2):
        d_lat, d_lg = torch.empty(R, 512, device=cuda), torch.empty(3, R, device=cuda)
        L.check(lib().neo_grid_encoder_pool_bwd_bf16(Lb.data_ptr(), 576, L.ptr(logits), nv, *[L.ptr(g) for g in ups], L.ptr(d_lat), L.ptr(d_lg),
                                                     None))
        runs.append((d_lat, d_lg))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
    d_lat32, d_lg32 = torch.empty(R, 512, device=cuda), torch.empty(3, R, device=cuda)
    L.check(lib().neo_grid_encoder_pool_bwd(L.ptr(lat), L.ptr(logits), nv, *[L.ptr(g) for g in ups], L.ptr(d_lat32), L.ptr(d_lg32), None))
    assert torch.equal(runs[0][0], d_lat32) and torch.equal(runs[0][1], d_lg32)
    mf = etm.pool_fwd(lat, logits, nv, G)
    mb = etm.pool_bwd(lat, logits, nv, G, *ups)
    errs = {n: tcm.rel_err(o, mf[n]) for n, o in zip(("xz", "xy", "yz"), out)}
    errs.update(d_lat=tcm.rel_err(runs[0][0], mb["d_lat"]), d_logits=tcm.rel_err(runs[0][1], mb["d_logits"]))
    print(f"pool bf16 nv={nv}: relative errors {json.dumps({k: float(f'{v:.3g}') for k, v in errs.items()})} (bound {tcm.POOL_BOUND})")
    assert max(errs.values()) <= tcm.POOL_BOUND


def dense_setup(dev, nv=1, seed=5):
    from neo360_b200.encoder import GridEncoder
    torch.manual_seed(seed)
    enc = GridEncoder(train_precision="tc").train().to(dev)
    lh, lw, W, H = 60, 80, 160, 120
    sc = synth.make_scene((W, H), 3, (4, 4), 1)
    poses, focal, c = sc["src_poses"][:nv].to(dev), sc["src_focal"][:nv].to(dev), sc["src_c"][:nv].to(dev)
    gen = torch.Generator().manual_seed(9)
    latent = (torch.rand(nv, 512, lh, lw, generator=gen) ** 2 * 2).to(dev)
    wts = [torch.randn(nv, 512, G, G, generator=gen).to(dev) for _ in range(3)]
    return enc, latent, (poses, focal, c, W, H), wts


def run_dense(enc, form, latent0, geo, wts):
    enc.zero_grad(set_to_none=True)
    latent = latent0.clone().requires_grad_(True)
    planes = getattr(enc, form)(latent, *geo)
    sum(((p * w).sum() for p, w in zip(planes, wts))).backward()
    grads = {n: p.grad.clone() for n, p in dense_params(enc).items()}
    grads["latent"] = latent.grad
    return [p.detach() for p in planes], grads


MODEL_NAMES = {"depth_fc.common_branch.0": "0", "depth_fc.common_branch.2": "1", "depth_fc.depth_encoder": "2"}


def model_name(n):
    """dense_params name -> the model's gradient name."""
    mod, kind = n.rsplit(".", 1)
    if mod in MODEL_NAMES:
        return ("w" if kind == "weight" else "b") + MODEL_NAMES[mod]
    axis, layer = mod.split(".")
    return f"{axis[4:]}_{'w' if kind == 'weight' else 'b'}{0 if layer == '0' else 1}"


def test_dense_part_matches_model_and_fp32(cuda):
    """NV = 1, latent 60 x 80: the three floor plans within FWD_BOUND and the latent and every parameter gradient within BWD_BOUND of
    the model at the kernels' rounding points (fed the fp32 entry's lookup rows); both within STEP_BOUND of the fp32 `dense_train`.  The
    second aggregator layers' bias gradients are exactly zero (shift_invariant) and are held to their weights' scale."""
    from neo360_b200 import _lib as L
    enc, latent0, geo, wts = dense_setup(cuda)
    planes, got = run_dense(enc, "dense_train_tc", latent0, geo, wts)
    ref_planes, ref = run_dense(enc, "dense_train", latent0, geo, wts)
    poses, focal, c, W, H = geo
    nv, _, lh, lw = latent0.shape
    R = nv * G ** 3
    # the model, float64 on the device, from the fp32 entry's lookup rows
    lat_cl = latent0.permute(0, 2, 3, 1).contiguous()
    pc = poses.float().contiguous()
    cam = (float(focal[0]), float(c[0, 0]), float(c[0, 1]))
    X = torch.empty(R, 520, device=cuda)
    L.check(lib().neo_grid_encoder_features(L.ptr(lat_cl), nv, lh, lw, W, H, L.ptr(pc), *cam, L.ptr(X), 520, None))
    with torch.no_grad():
        mp, _, S = tcm.forward(X, tcm.grid_coords(G, nv, device=cuda), tcm.params_of(enc), nv, G)
        del X
        mb = tcm.backward(wts[0].double(), wts[1].double(), wts[2].double(), S, tcm.params_of(enc), nv, G)
        del S
    g_lat = torch.zeros(nv, lh, lw, 512, device=cuda)
    gx = mb.pop("g_X").float().contiguous()
    L.check(lib().neo_grid_encoder_features_bwd(nv, lh, lw, W, H, L.ptr(pc), *cam, L.ptr(gx), 512, L.ptr(g_lat), None))
    errs = {f"plane_{n}": tcm.rel_err(p, mp[n]) for n, p in zip(("xz", "xy", "yz"), planes)}
    assert max(errs.values()) <= tcm.FWD_BOUND, errs
    zero = shift_invariant(enc)
    berrs = {"latent": tcm.rel_err(got["latent"], g_lat.permute(0, 3, 1, 2))}
    for n, g in got.items():
        if n == "latent":
            continue
        m = mb[model_name(n)]
        if n in zero:
            w = mb[model_name(n[:-len("bias")] + "weight")]
            assert float((g.double() - m).abs().max()) <= tcm.BWD_BOUND * float(w.abs().max()), n
            continue
        berrs[n] = tcm.rel_err(g, m)
    print("dense tc vs model: forward", json.dumps({k: float(f"{v:.3g}") for k, v in errs.items()}), "backward",
          json.dumps({k: float(f"{v:.3g}") for k, v in sorted(berrs.items(), key=lambda kv: -kv[1])}))
    assert max(berrs.values()) <= tcm.BWD_BOUND, berrs
    serrs = {f"plane_{i}": tcm.rel_err(p, r) for i, (p, r) in enumerate(zip(planes, ref_planes))}
    serrs.update({n: tcm.rel_err(got[n], ref[n]) for n in ref if n not in zero})
    print("dense tc vs fp32 dense_train:", json.dumps({k: float(f"{v:.3g}") for k, v in sorted(serrs.items(), key=lambda kv: -kv[1])[:8]}))
    assert max(serrs.values()) <= tcm.STEP_BOUND, serrs


def fold_biases(grads, names):
    """A bias whose exact gradient is zero or one nearly cancelling scalar is held to the bound together with its weight's gradient."""
    for b in [k for k in grads if k in names]:
        w = b[:-len("bias")] + "weight"
        grads[w] = torch.cat([grads[w].reshape(-1), grads.pop(b).reshape(-1)])
    return grads


def test_training_step_with_tc_encoder(cuda):
    """The NeO-360 training step of BASELINE configs[3] (4096 rays, 128 + 64 samples, 3 source views of 640 x 480) with the encoder
    inside it, `train_precision="tc"` on both the renderer and the encoder: every parameter's gradient within ENC_STEP_BOUND of the
    all-fp32 step (biases without a signal of their own folded into their weights)."""
    from neo360_b200 import NeRF_TP, batches
    from neo360_b200.encoder import GridEncoder
    from neo360_b200.training import training_loss
    sc = synth.make_scene((640, 480), 3, (120, 160), 0)
    g0 = torch.Generator().manual_seed(77)
    src = {"src_poses": sc["src_poses"].to(cuda), "src_focal": sc["src_focal"].to(cuda), "src_c": sc["src_c"].to(cuda),
           "src_imgs": (torch.rand(3, 3, 480, 640, generator=g0) * 2 - 1).to(cuda)}
    g = torch.Generator().manual_seed(1234)
    tposes = torch.stack([synth.target_pose(5 * k, 100)[:3, :4] for k in range(batches.NUM_TARGET_VIEWS)]).to(cuda)
    views = batches.TargetViews(tposes, torch.rand(batches.NUM_TARGET_VIEWS, 480, 640, 3, generator=g).to(cuda), 0.8 * 640)
    batch = batches.train_batch(views, src, pix_inds=batches.draw_pix_inds(views.T, views.H, views.W, 4096, g))
    grads = {}
    for prec in ("fp32", "tc"):
        torch.manual_seed(0)
        net = NeRF_TP(num_coarse_samples=128, num_fine_samples=64, num_src_views=3, precision="fp32",
                      encoder=GridEncoder(train_precision=prec), train_precision=prec)
        sd = net.state_dict()
        sd.update(synth.make_mlp_params(0))
        net.load_state_dict(sd)
        net = net.to(cuda).train()
        torch.manual_seed(1)
        ret = net(batch, True, False, None, None)
        training_loss(ret, batch["target"]).backward()
        names = shift_invariant(net.encoder, "encoder.") | {n for n, _ in net.named_parameters() if n.endswith("density_layer.bias")}
        grads[prec] = fold_biases({n: p.grad.clone() for n, p in net.named_parameters() if p.grad is not None}, names)
        del net, ret
        torch.cuda.empty_cache()
    assert set(grads["tc"]) == set(grads["fp32"]) and any(n.startswith("encoder.depth_fc") for n in grads["tc"])
    errs = {n: tcm.rel_err(grads["tc"][n], grads["fp32"][n]) for n in grads["fp32"]}
    print("training step, renderer and encoder tc vs fp32:", json.dumps({k: round(v, 5) for k, v in sorted(errs.items(), key=lambda kv: -kv[1])[:10]}))
    assert max(errs.values()) <= tcm.ENC_STEP_BOUND, errs


def test_convergence(cuda):
    """Teacher / student on the dense part (NV = 1, latent 60 x 80): the teacher's planes (parameters seed 1, fp32 inference) are the
    target; the student (seed 5) takes 300 Adam steps on depth_fc and the aggregators with the fp32 and with the tc form.  Measured on
    an H100 80GB HBM3 at 700 W: final loss 0.0165396 (tc) against 0.0166034 (fp32), from 1.0257; the a-priori bound is 10 %."""
    from neo360_b200.encoder import GridEncoder
    _, latent, geo, _ = dense_setup(cuda)
    torch.manual_seed(1)
    teacher = GridEncoder().to(cuda).eval()
    with torch.no_grad():
        target = teacher.dense_cuda(latent, *geo)
    curves = {}
    for form in ("dense_train", "dense_train_tc"):
        torch.manual_seed(5)
        enc = GridEncoder().to(cuda).train()
        params = list(dense_params(enc).values())
        opt = torch.optim.Adam(params, lr=1e-4)
        losses = []
        for _ in range(300):
            planes = getattr(enc, form)(latent, *geo)
            loss = sum(((p - t) ** 2).mean() for p, t in zip(planes, target))
            opt.zero_grad(set_to_none=True)
            loss.backward()
            opt.step()
            losses.append(float(loss.detach()))
        curves[form] = losses
    print("convergence", json.dumps({k: [float(f"{v[i]:.6g}") for i in (0, 100, 200, 299)] for k, v in curves.items()}))
    f32, tc = curves["dense_train"], curves["dense_train_tc"]
    assert f32[-1] < f32[0] and tc[-1] < tc[0]
    assert abs(tc[-1] - f32[-1]) <= 0.1 * f32[-1]


DET_SCRIPT = r"""
import json, sys, torch
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[1] + "/tests")
torch.use_deterministic_algorithms(True)
from test_gpu_encoder_train_tc import dense_setup, dense_params
dev = torch.device("cuda:0")
out = []
for run in range(2):
    enc, latent0, geo, wts = dense_setup(dev)
    params = list(dense_params(enc).values())
    latent = latent0.clone().requires_grad_(True)
    opt = torch.optim.Adam(params + [latent], lr=1e-4)
    rec = []
    for s in range(3):
        planes = enc.dense_train_tc(latent, *geo)
        loss = sum(((p * w).sum() for p, w in zip(planes, wts)))
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
        rec.append(loss.item())
    state = [t.detach().reshape(-1).cpu() for p in params + [latent] for t in (p, opt.state[p]["exp_avg"], opt.state[p]["exp_avg_sq"])]
    out.append((rec, torch.cat(state)))
print(json.dumps({"losses": out[0][0] == out[1][0], "state": torch.equal(out[0][1], out[1][1])}))
"""


def test_deterministic_steps(cuda):
    """Three Adam steps on the dense part and the latent, twice, under torch.use_deterministic_algorithms(True) in a subprocess:
    bit-identical losses, parameters and Adam state."""
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    res = subprocess.run([sys.executable, "-c", DET_SCRIPT, ROOT], capture_output=True, text=True, env=env, timeout=900)
    assert res.returncode == 0, res.stderr[-3000:]
    r = json.loads(res.stdout.strip().splitlines()[-1])
    assert r == {"losses": True, "state": True}, r


def test_inference_unchanged_by_train_precision(cuda):
    """After a tc training step, the encoder's inference output equals that of an fp32 encoder loaded with its state dict, bit for bit."""
    from neo360_b200.encoder import GridEncoder
    torch.manual_seed(8)
    tc = GridEncoder(train_precision="tc").to(cuda).train()
    sc = synth.make_scene((160, 120), 1, (4, 4), 3)
    gen = torch.Generator().manual_seed(12)
    imgs = (torch.rand(1, 3, 120, 160, generator=gen) * 2 - 1).to(cuda)
    args = (imgs, sc["src_poses"].to(cuda), sc["src_focal"].to(cuda), sc["src_c"].to(cuda))
    opt = torch.optim.Adam(tc.parameters(), lr=1e-4)
    sum(o.square().mean() for o in tc(*args)).backward()
    opt.step()
    ref = GridEncoder().to(cuda)
    ref.load_state_dict(tc.state_dict())
    tc.eval(), ref.eval()
    with torch.no_grad():
        a, b = tc(*args), ref(*args)
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_default_path_is_dense_train(cuda):
    """With the default train_precision ("fp32") the training forward runs `dense_train` and never the tc form; with "tc" the reverse."""
    from neo360_b200.encoder import GridEncoder
    torch.manual_seed(9)
    enc = GridEncoder().to(cuda).train()
    assert enc.train_precision == "fp32"
    sc = synth.make_scene((160, 120), 1, (4, 4), 3)
    imgs = (torch.rand(1, 3, 120, 160, generator=torch.Generator().manual_seed(13)) * 2 - 1).to(cuda)
    args = (imgs, sc["src_poses"].to(cuda), sc["src_focal"].to(cuda), sc["src_c"].to(cuda))
    calls = []
    for name in ("dense_train", "dense_train_tc"):
        fn = getattr(enc, name)
        setattr(enc, name, lambda *a, fn=fn, name=name: calls.append(name) or fn(*a))
    enc(*args)
    enc.train_precision = "tc"
    enc(*args)
    assert calls == ["dense_train", "dense_train_tc"]
    with pytest.raises(ValueError, match="train_precision"):
        enc.train_precision = "bogus"
    with pytest.raises(ValueError, match="train_precision"):
        GridEncoder(train_precision="bogus")
