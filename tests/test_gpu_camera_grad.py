"""GPU: ray and pose gradients of vanilla NeRF (pose refinement).

* per ray: `neo_vanilla_encode_bwd` against the float64 model (oracle/camera_grad_model.py) at the kernel's own fp32 points, every ray
  within ENC_K N 2^-24 sum|terms|; `neo_sample_rays_bwd` against the float64 model per view within RAYS_K n_view 2^-24 sum|terms|;
* end to end against tests/golden/camera_grad_vectors.npz (the reference NeRF in float64 under autograd): outputs and ray gradients of
  `NeRF.forward` with the MLP frozen, train_precision fp32 and tc, and the pose gradient through `ops.sample_rays`;
* a graph to the rays exists with the MLP frozen and in eval mode; radii and target carry none;
* the same training step with and without rays requiring grad gives bit-identical outputs and parameter gradients;
* two runs give bit-identical ray and pose gradients;
* a short pose refinement (tools/refine_poses.py) brings both pose errors below REFINE_FRACTION of their start;
* `_MLPTrainTC`'s input-row gradient against the float64 model at its bf16 rounding points (oracle/camera_grad_model.mlp_input_grad);
* Mip-NeRF 360: `neo_mip_composite_bwd_rays_d` per ray against float64 autograd, and end to end against the fixture (viewdirs and rays_d
  get the reference's gradients, rays_o and radii none, as the reference's detached contract gives), no bit of training changed.
Run with `-m gpu -s` to see the measured values."""
import importlib.util
import os

import numpy as np
import pytest
import torch

from oracle import camera_grad_model as cgm

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "camera_grad_vectors.npz")
U = 2.0 ** -24
ENC_K = 4.0
RAYS_K = 4.0
E2E_OUT = 2e-4            # outputs vs the float64 reference, as tests/test_gpu_vanilla_train.py's tuples
# relative L2 errors of each ray gradient and of g_c2w against the float64 reference, about 2.5x the values measured on an H100 80GB HBM3
# at 700 W: fp32 3.7e-3 (rays_o) and 4.0e-3 (c2w): the fp32 points and sample positions, through sin(2^9 x); tc 0.22 and 0.12: the bf16
# activations and data gradients of eight layers (the tc path's parameter gradients carry the same bf16 error).  The tc input-row gradient
# itself is held to the dense chain's model bound by test_mlp_input_grad_against_model.
E2E_GRAD = {"fp32": 1e-2, "tc": 0.5}
POSE_GRAD = {"fp32": 1e-2, "tc": 0.3}
# relative L2 of Mip-NeRF 360's g_viewdirs and g_rays_d against the float64 reference: measured 6.9e-7 (fp32) and 2.3e-2 (tc, viewdirs) on an
# H100 80GB HBM3 at 700 W
MIP_GRAD = {"fp32": 1e-5, "tc": 6e-2}
REFINE_FRACTION = 0.5


@pytest.fixture(scope="module")
def cuda():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from neo360_b200 import build
    build.build()
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def gold():
    return {k: torch.from_numpy(v) if v.dtype != object else v for k, v in np.load(GOLD).items()}


def rel(a, b):
    return float((a.double().cpu() - b.double()).norm() / b.double().norm())


def frozen_net(gold, prec, dev):
    from neo360_b200 import synth
    from neo360_b200.vanilla import NeRF
    W, H, B, nc, nf, seed = [int(x) for x in gold["cfg"]]
    net = NeRF(num_coarse_samples=nc, num_fine_samples=nf, train_precision=prec)
    net.load_state_dict(synth.make_vanilla_params(seed))
    return net.to(dev).eval().requires_grad_(False)


def loss_of(ret, gold, dev):
    return sum((ret[l][0] * gold[f"g_rgb{l}"].float().to(dev)).sum() + (ret[l][1] * gold[f"g_acc{l}"].float().to(dev)).sum() for l in range(2))


def test_encode_bwd_per_ray(cuda):
    from neo360_b200 import _lib as L
    lib = L.load()
    g = torch.Generator().manual_seed(3)
    for n, N in ((1, 1), (37, 33), (300, 129)):
        o = torch.rand(n, 3, generator=g) * 2 - 1
        vd = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1)
        vd[0] *= 1.7                                         # viewdirs of any length
        t = torch.sort(torch.rand(n, N, generator=g) * 2.8 + 0.2, -1).values
        ge, gd = torch.randn(n * N, 63, generator=g), torch.randn(n, 27, generator=g)
        out = [torch.empty(n, 3, device=cuda) for _ in range(2)]
        dv = [x.to(cuda).contiguous() for x in (o, vd, t, ge, gd)]
        L.check(lib.neo_vanilla_encode_bwd(*[L.ptr(x) for x in dv[:3]], n, N, L.ptr(dv[3]), L.ptr(dv[4]), L.ptr(out[0]), L.ptr(out[1]),
                                           torch.cuda.current_stream().cuda_stream))
        x32 = o[:, None, :] + t[..., None] * vd[:, None, :]          # the kernel's fp32 points: one rounded multiply, one rounded add
        g_o, g_vd, m_o, m_vd = cgm.vanilla_encode_bwd(o.double(), vd.double(), t.double(), ge.double(), gd.double(), x=x32.double())
        eo = ((out[0].cpu().double() - g_o).abs() / (N * U * m_o)).max()
        ev = ((out[1].cpu().double() - g_vd).abs() / ((N + 1) * U * m_vd)).max()
        print(f"encode_bwd n={n} N={N}: max error / (N 2^-24 sum|terms|) = {float(eo):.3f} (rays_o), {float(ev):.3f} (viewdirs)")
        assert float(eo) <= ENC_K and float(ev) <= ENC_K


def test_sample_rays_bwd_per_view(cuda):
    from neo360_b200 import ops, synth
    T, H, W, f, n = 3, 48, 64, 51.2, 4096
    g = torch.Generator().manual_seed(5)
    c2w = torch.stack([synth.target_pose(9 * k, 100)[:3, :4] for k in range(T)]).to(cuda)
    pix = torch.randint(0, T * H * W, (n,), generator=g).to(cuda)
    with torch.no_grad():
        ref = ops.sample_rays(pix, H, W, f, c2w)
    leaf = c2w.clone().requires_grad_(True)
    o, vd, rd, rad, tgt = ops.sample_rays(pix, H, W, f, leaf)
    for a, b in zip((o, vd, rd, rad), ref):
        assert torch.equal(a, b)                                      # forward bits unchanged
    assert not rad.requires_grad and tgt is None
    go, gv, gr = (torch.randn(n, 3, generator=g) for _ in range(3))
    ((o * go.to(cuda)).sum() + (vd * gv.to(cuda)).sum() + (rd * gr.to(cuda)).sum()).backward()
    want, mag = cgm.sample_rays_bwd(pix.cpu(), T, H, W, f, c2w.cpu().double(), go.double(), gv.double(), gr.double())
    counts = torch.bincount(pix.cpu() // (H * W), minlength=T).double()[:, None, None]
    err = ((leaf.grad.cpu().double() - want).abs() / (counts * U * mag + 1e-30)).max()
    print(f"sample_rays_bwd: max error / (n_view 2^-24 sum|terms|) = {float(err):.3f}")
    assert float(err) <= RAYS_K
    first = leaf.grad.clone()
    leaf.grad = None
    o, vd, rd, _, _ = ops.sample_rays(pix, H, W, f, leaf)
    ((o * go.to(cuda)).sum() + (vd * gv.to(cuda)).sum() + (rd * gr.to(cuda)).sum()).backward()
    assert torch.equal(first, leaf.grad)                               # deterministic
    # get_rays: the frame's rays, differentiable the same way
    leaf1 = c2w[1].clone().requires_grad_(True)
    o1, v1, r1, rad1 = ops.get_rays(H, W, f, leaf1)
    with torch.no_grad():
        ref1 = ops.get_rays(H, W, f, c2w[1])
    assert all(torch.equal(a, b) for a, b in zip((o1, v1, r1, rad1), ref1))
    v1.sum().backward()
    assert leaf1.grad is not None and bool(torch.isfinite(leaf1.grad).all())


@pytest.mark.parametrize("prec", ["fp32", "tc"])
def test_ray_gradients_vs_reference(cuda, gold, prec):
    net = frozen_net(gold, prec, cuda)
    near, far = [float(x) for x in gold["near_far"]]
    rays = {k: gold[f"rays_{k}"].float().to(cuda).requires_grad_(True) for k in ("rays_o", "rays_d", "viewdirs")}
    ret = net(rays, False, True, near, far)
    assert ret[1][0].grad_fn is not None                              # frozen MLP, eval mode: a graph to the rays
    for l in range(2):
        e = max(float((ret[l][0].detach().cpu().double() - gold[f"rays_rgb{l}"]).abs().max()),
                float((ret[l][1].detach().cpu().double() - gold[f"rays_acc{l}"]).abs().max()))
        print(f"[{prec}] level {l}: outputs max|diff| {e:.2e}")
        assert e < (E2E_OUT if prec == "fp32" else 3e-2)
    loss_of(ret, gold, cuda).backward()
    for k in ("rays_o", "rays_d", "viewdirs"):
        r = rel(rays[k].grad, gold[f"rays_g_{k}"])
        print(f"[{prec}] g_{k}: relative L2 error {r:.2e}")
        assert r < E2E_GRAD[prec]


@pytest.mark.parametrize("prec", ["fp32", "tc"])
def test_pose_gradient_vs_reference(cuda, gold, prec):
    from neo360_b200 import ops
    net = frozen_net(gold, prec, cuda)
    W, H = int(gold["cfg"][0]), int(gold["cfg"][1])
    near, far = [float(x) for x in gold["near_far"]]
    c2w = gold["pose"].float().to(cuda)[None].requires_grad_(True)
    o, vd, rd, rad, _ = ops.sample_rays(gold["sel"].long().to(cuda), H, W, float(gold["focal"]), c2w)
    ret = net({"rays_o": o, "rays_d": rd, "viewdirs": vd, "radii": rad}, False, True, near, far)
    loss_of(ret, gold, cuda).backward()
    r = rel(c2w.grad[0], gold["pose_g_c2w"])
    print(f"[{prec}] g_c2w: relative L2 error {r:.2e}")
    assert r < POSE_GRAD[prec]


@pytest.mark.parametrize("prec", ["fp32", "tc"])
def test_ray_grad_changes_no_bit_of_training(cuda, gold, prec):
    """A training step with rays that require grad gives the same outputs and parameter gradients, bit for bit, as without."""
    from neo360_b200 import synth
    from neo360_b200.vanilla import NeRF
    near, far = [float(x) for x in gold["near_far"]]
    res = []
    for ray_grad in (False, True):
        torch.manual_seed(0)
        net = NeRF(num_coarse_samples=32, num_fine_samples=32, train_precision=prec)
        net.load_state_dict(synth.make_vanilla_params(1))
        net = net.to(cuda).train()
        rays = {k: gold[f"rays_{k}"].float().to(cuda).requires_grad_(ray_grad) for k in ("rays_o", "rays_d", "viewdirs")}
        u = [torch.rand(rays["rays_o"].shape[0], n, device=cuda, generator=torch.Generator(device=cuda).manual_seed(n)) for n in (33, 32)]
        ret = net({**rays, "_uniforms": u}, True, True, near, far)
        loss_of(ret, gold, cuda).backward()
        res.append(([t.detach().clone() for lv in ret for t in lv], [p.grad.clone() for p in net.parameters()]))
    for a, b in zip(res[0][0] + res[0][1], res[1][0] + res[1][1]):
        assert torch.equal(a, b)


def test_ray_and_pose_gradients_are_deterministic(cuda, gold):
    from neo360_b200 import ops
    net = frozen_net(gold, "fp32", cuda)
    W, H = int(gold["cfg"][0]), int(gold["cfg"][1])
    near, far = [float(x) for x in gold["near_far"]]
    runs = []
    for _ in range(2):
        c2w = gold["pose"].float().to(cuda)[None].requires_grad_(True)
        o, vd, rd, _, _ = ops.sample_rays(gold["sel"].long().to(cuda), H, W, float(gold["focal"]), c2w)
        leaves = [x.detach().requires_grad_(True) for x in (o, vd, rd)]
        ret = net(dict(zip(("rays_o", "viewdirs", "rays_d"), leaves)), False, True, near, far)
        loss_of(ret, gold, cuda).backward()
        torch.autograd.backward([o, vd, rd], [x.grad for x in leaves])
        runs.append([x.grad.clone() for x in leaves] + [c2w.grad.clone()])
    for a, b in zip(*runs):
        assert torch.equal(a, b)


def test_pose_refinement_recovers_perturbed_poses(cuda):
    spec = importlib.util.spec_from_file_location("refine_poses", os.path.join(ROOT, "tools", "refine_poses.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    before, after = mod.refine(steps=150, log=print)
    print(f"pose refinement: rotation {before[0]:.4f} -> {after[0]:.4f} deg, translation {before[1]:.5f} -> {after[1]:.5f}")
    assert after[0] < REFINE_FRACTION * before[0] and after[1] < REFINE_FRACTION * before[1]


@pytest.mark.parametrize("kind,n,N", [("vanilla", 1037, 65), ("prop", 2048, 64), ("mip", 517, 32)])
def test_mlp_input_grad_against_model(cuda, kind, n, N):
    """`_MLPTrainTC`'s input-row gradient (layer 0's and the skip layer's feature columns, bf16 GEMMs with fp32 epilogues, added in fp32)
    within the dense chain's backward bound of the float64 model at its bf16 rounding points (oracle/camera_grad_model.mlp_input_grad over
    oracle/dense_train_model.py); the model with half of the skip term lies beyond twice that bound."""
    from neo360_b200 import mip, training, vanilla
    from oracle import dense_train_model as dtm
    torch.manual_seed(3)
    m, F = (vanilla.NeRFMLP(), 63) if kind == "vanilla" else ((mip.PropMLP(), 504) if kind == "prop" else (mip.NeRFMLP(), 504))
    g = torch.Generator().manual_seed(3)
    with torch.no_grad():
        for p in m.parameters():
            p.add_(0.01 * torch.randn(p.shape, generator=g))
    m = m.to(cuda)
    M = n * N
    feats = torch.randn(M, F, generator=g).clamp(-1, 1).to(cuda).requires_grad_(True)
    gs = (torch.randn(M, 1, generator=g) * 1e-3).to(cuda)
    gy = (torch.randn(M, 128, generator=g) * 1e-3).to(cuda)
    layers = m.pts_linears if hasattr(m, "pts_linears") else m.pts_linear
    params = [t for lin in layers for t in (lin.weight, lin.bias)] + [m.density_layer.weight, m.density_layer.bias]
    if hasattr(m, "rgb_layer"):
        params += [m.bottleneck_layer.weight, m.bottleneck_layer.bias, m.views_linear[0].weight[:, :256]]
        sig, yb = training._MLPTrainTC.apply(len(layers), feats, *params)
        ((sig * gs).sum() + (yb * gy).sum()).backward()
    else:
        yb, gy = None, None
        (training._MLPTrainTC.apply(len(layers), feats, *params) * gs).sum().backward()
    P = dtm.params_of(m)
    _, _, S = dtm.forward(feats.detach().double(), P)
    want = cgm.mlp_input_grad(gs.double(), None if gy is None else gy.double(), S, P, F)
    err = dtm.rel_err(feats.grad, want)
    bound = dtm.WIDE_BWD_BOUND if kind == "mip" else dtm.BWD_BOUND
    print(f"_MLPTrainTC input-row gradient {kind} {n}x{N}: {err:.2e} of the model (bound {bound})")
    assert err < bound
    if len(P["w"]) > 5:
        assert dtm.rel_err(cgm.mlp_input_grad(gs.double(), gy.double(), S, P, F, skip_scale=0.5), want) > 2 * bound


def test_mip_composite_rays_d_per_ray(cuda):
    """neo_mip_composite_bwd_rays_d: the same d_raw_density / d_raw_rgb bits as neo_mip_composite_bwd, and g_rays_d equal to float64
    autograd through oracle/mip_train_model.composite_fwd w.r.t. rays_d."""
    from neo360_b200 import _lib as L
    from oracle import mip_train_model as mtm
    lib = L.load()
    g = torch.Generator().manual_seed(9)
    n, N = 300, 33
    rd = torch.randn(n, N, generator=g) * 2
    rc = torch.randn(n, N, 3, generator=g)
    t = torch.sort(torch.rand(n, N + 1, generator=g) * 5.8 + 0.2, -1).values
    d = torch.randn(n, 3, generator=g) * 1.5
    g_rgb, g_w = torch.randn(n, 3, generator=g), torch.randn(n, N, generator=g)
    dv = [x.to(cuda).contiguous() for x in (rd, rc, t, d, g_rgb, g_w)]
    outs = [[torch.empty(n, N, device=cuda), torch.empty(n, N, 3, device=cuda)] for _ in range(2)]
    g_d = torch.empty(n, 3, device=cuda)
    s = torch.cuda.current_stream().cuda_stream
    P = L.ptr
    L.check(lib.neo_mip_composite_bwd(P(dv[0]), P(dv[1]), P(dv[2]), P(dv[3]), n, N, P(dv[4]), P(dv[5]), None, None, P(outs[0][0]), P(outs[0][1]), s))
    L.check(lib.neo_mip_composite_bwd_rays_d(P(dv[0]), P(dv[1]), P(dv[2]), P(dv[3]), n, N, P(dv[4]), P(dv[5]), None, None, P(outs[1][0]),
                                             P(outs[1][1]), P(g_d), s))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    dd = d.double().requires_grad_(True)
    o = mtm.composite_fwd(rd.double(), rc.double(), t.double(), dd, fp32=False)
    ((o["rgb"] * g_rgb.double()).sum() + (o["w"] * g_w.double()).sum()).backward()
    r = rel(g_d, dd.grad)
    print(f"mip g_rays_d: relative L2 error {r:.2e}")
    assert r < 1e-4


def mip_net(prec, dev):
    from neo360_b200 import synth
    from neo360_b200.mip import MipNeRF360
    net = MipNeRF360(num_prop_samples=16, num_nerf_samples=8, train_precision=prec)
    net.load_state_dict(synth.make_mip_params(0))
    return net.to(dev)


def mip_loss(ren, hist, gold, dev):
    return (ren[2]["rgb"] * gold["mip_g_rgb"].float().to(dev)).sum() + sum((hist[l]["weights"] * gold[f"mip_g_w{l}"].float().to(dev)).sum()
                                                                          for l in range(3))


@pytest.mark.parametrize("prec", ["fp32", "tc"])
def test_mip_ray_gradients_vs_reference(cuda, gold, prec):
    """Mip-NeRF 360 with the MLPs frozen: viewdirs (direction encoding) and rays_d (|rays_d| in the compositing) get the reference's
    gradients; rays_o and radii get none, as in the reference, whose contract detaches the Gaussians."""
    net = mip_net(prec, cuda).eval().requires_grad_(False)
    near, far = float(gold["mip_cfg"][2]), float(gold["mip_cfg"][3])
    batch = {k: gold[f"mip_{k}"].float().to(cuda).requires_grad_(True) for k in ("rays_o", "rays_d", "viewdirs", "radii")}
    ren, hist = net(batch, 1.0, False, False, near, far)
    e = float((ren[2]["rgb"].detach().cpu().double() - gold["mip_rgb2"]).abs().max())
    print(f"[mip {prec}] rgb max|diff| {e:.2e}")
    assert e < (5e-4 if prec == "fp32" else 3e-2)
    mip_loss(ren, hist, gold, cuda).backward()
    assert batch["rays_o"].grad is None and batch["radii"].grad is None
    assert bool((gold["mip_g_rays_o"] == 0).all()) and bool((gold["mip_g_radii"] == 0).all())
    for k in ("rays_d", "viewdirs"):
        r = rel(batch[k].grad, gold[f"mip_g_{k}"])
        print(f"[mip {prec}] g_{k}: relative L2 error {r:.2e}")
        assert r < MIP_GRAD[prec]


@pytest.mark.parametrize("prec", ["fp32", "tc"])
def test_mip_ray_grad_changes_no_bit_of_training(cuda, gold, prec):
    near, far = float(gold["mip_cfg"][2]), float(gold["mip_cfg"][3])
    res = []
    for ray_grad in (False, True):
        net = mip_net(prec, cuda).train()
        batch = {k: gold[f"mip_{k}"].float().to(cuda).requires_grad_(ray_grad) for k in ("rays_o", "rays_d", "viewdirs", "radii")}
        ren, hist = net(batch, 1.0, False, True, near, far)
        mip_loss(ren, hist, gold, cuda).backward()
        res.append(([r["rgb"].detach().clone() for r in ren] + [h["weights"].detach().clone() for h in hist],
                    [p.grad.clone() if p.grad is not None else torch.zeros(0) for p in net.parameters()]))
    for a, b in zip(res[0][0] + res[0][1], res[1][0] + res[1][1]):
        assert torch.equal(a, b)
