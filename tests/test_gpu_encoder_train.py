"""GPU: the GridEncoder training path (`GridEncoder.dense_train`: `neo_grid_encoder_features(_bwd)`, `neo_grid_encoder_pool(_bwd)` and
framework fp32 GEMMs) stage by stage against the float64 model (oracle/encoder_train_model.py, pinned to autograd through `dense_torch`
on the CPU by tests/test_encoder_train_model.py), and end to end against autograd through `dense_torch`.

Bounds: the constants below, 2-3x the maxima measured on an H100 (DESIGN.md section 2 lists the card, its power limit and the measured
values).  Run with `-m gpu -s`: every comparison prints its measured maximum.
"""
import copy
import gc

import pytest
import torch

from neo360_b200 import synth
from oracle import encoder_train_model as etm
from oracle import tc_paths_model as tpm
from test_gpu_tc_paths import encoder_poses

pytestmark = pytest.mark.gpu

G = 64
U = 2.0 ** -24
# lookup rows: |X - model| <= FEAT_TOL * sum |w F| + 2 derr (columns 0..511; measured: within 2 derr everywhere); cam / direction
# columns absolute (measured 1.1e-7)
FEAT_TOL, FEAT_GEO_TOL = 8 * U, 1e-5
# lookup adjoint per texel: |g_lat - model| <= FEAT_BWD_TOL * n * sum |w g| + 2 derr (n = contributions: unordered fp32 atomics;
# measured: within 2 derr everywhere)
FEAT_BWD_TOL = 4 * U
# pool forward / backward in units of their magnitudes (sum of the absolute terms): (POOL_TOL + POOL_SPREAD_TOL x spread) 2^-24, spread
# = the largest |logit - pillar max| of a contributing cell (measured 13.3 forward, 15.5 backward at spread <= 2, 73.4 at spread 80)
POOL_TOL, POOL_SPREAD_TOL, FLOOR = 32, 2, 8 * 2.0 ** -149
# end to end, per gradient tensor: max error <= E2E_MAX of its largest |reference| and relative L2 <= E2E_L2 (measured 1.8e-2 / 2.9e-3
# against float64, 1.0e-2 / 2.8e-3 in the training step).  The largest errors are in the latent and the aggregators' first-layer
# weights, sums over the 64^3 x NV grid rows of fp32 GEMM products.  The fp32-against-fp32 comparison at the production shape carries
# both forms' rounding through the ResNet and the conv stacks as well (measured 2.9e-2 / 7.0e-3).
E2E_MAX, E2E_L2, E2E_FP32_MAX, E2E_FP32_L2 = 5e-2, 8e-3, 7e-2, 1.5e-2


@pytest.fixture(scope="module")
def cuda():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from neo360_b200 import build
    build.build()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    return torch.device("cuda:0")


@pytest.fixture(autouse=True)
def release_memory():
    """The production-shape cases need most of the card: return what the previous case left cached."""
    yield
    gc.collect()
    torch.cuda.empty_cache()


def lib():
    from neo360_b200 import _lib as L
    return L.load()


def geometry(nv, lat_hw):
    lh, lw = lat_hw
    W, H = 2 * lw, 2 * lh
    poses = encoder_poses(nv)
    focal = torch.full((nv,), 0.8 * W)
    c = torch.tensor([[W / 2.0, H / 2.0]] * nv)
    return poses, focal, c, W, H


def ill_rows(nv, lat_hw, poses, focal, c, W, H, dev):
    """Rows whose mask or projection is ill-conditioned in fp32 (as tests/test_gpu_tc_paths.py leaves them out)."""
    _, cam, _, uv = tpm.encoder_geometry(etm._cells(G, nv), G, poses.double().to(dev), float(focal[0]), c[0].double(), W, H, lat_hw)
    z = cam[..., 2].reshape(-1)
    uv = uv.reshape(-1, 2)
    return ((z - 1e-3).abs() < 1e-5) | ((z.abs() < 1e-4) & (uv.abs().amax(-1) < 1e3))


@pytest.mark.parametrize("nv,lat_hw", [(1, (11, 18)), (3, (19, 12)), (8, (11, 18)), (3, (240, 320))])
def test_features_match_model(cuda, nv, lat_hw):
    """Lookup rows and their adjoint against the model at the kernel's fp32 tap coordinates, cameras with cells behind them, on
    z_cam = 0 and projecting outside the latent.  Ill-conditioned rows are left out of the forward and get a zero row gradient.  The
    gradient map starts from a sentinel: texels no row reaches stay bit-identical."""
    from neo360_b200 import _lib as L
    poses, focal, c, W, H = geometry(nv, lat_hw)
    lh, lw = lat_hw
    R = nv * G ** 3
    gen = torch.Generator().manual_seed(nv + lh)
    lat_cl = (torch.rand(nv, lh, lw, 512, generator=gen) * 4 - 1).to(cuda)
    pc = poses.float().contiguous().to(cuda)
    X = torch.empty(R, 520, device=cuda)
    geo = (nv, lh, lw, W, H)
    cam_args = (float(focal[0]), float(c[0, 0]), float(c[0, 1]))
    L.check(lib().neo_grid_encoder_features(L.ptr(lat_cl), *geo, L.ptr(pc), *cam_args, L.ptr(X), 520, None))
    tp, cam, dvec = etm.features_taps(G, lat_hw, poses.to(cuda), float(focal[0]), c[0], W, H)
    ill = ill_rows(nv, lat_hw, poses, focal, c, W, H, cuda)
    keep = ~ill
    m = etm.features_fwd(lat_cl.permute(0, 3, 1, 2), tp, cam, dvec)
    geo_err = float((X[:, 512:518].double() - m["X"][:, 512:]).abs()[keep].max())
    err = (X[:, :512].double() - m["X"][:, :512]).abs_()
    del m["X"]
    err.sub_(m["derr"].mul_(2))
    ok = bool((err <= FEAT_TOL * m["mag"])[keep].all())
    rel = float((err / m["mag"].clamp(min=1e-30))[keep].max()) / U
    del err, m
    print(f"features nv={nv} latent {lh}x{lw}: {int(ill.sum())} of {R} rows left out; lookup max (|err| - 2 derr) / sum|wF| "
          f"{rel:.2f} x 2^-24, cam/dir max {geo_err:.2e}")
    assert ok and geo_err <= FEAT_GEO_TOL
    assert bool(((X[:, 518:] == 0).all()))
    # adjoint
    g = torch.randn(R, 518, generator=gen).to(cuda)
    g[ill] = 0
    m = etm.features_bwd(tp, g, nv)
    for start in (0.0, -3.0):
        g_lat = torch.full((nv, lh, lw, 512), start, device=cuda)
        L.check(lib().neo_grid_encoder_features_bwd(*geo, L.ptr(pc), *cam_args, L.ptr(g), 518, L.ptr(g_lat), None))
        if start == 0.0:
            err = (g_lat.double() - m["val"]).abs()
            n = m["n"][..., None].clamp(min=1)
            bound = FEAT_BWD_TOL * n * m["mag"] + 2 * m["derr"]
            rel = (err - 2 * m["derr"]) / (n * m["mag"]).clamp(min=1e-30) / U
            print(f"features bwd nv={nv} latent {lh}x{lw}: max (|err| - 2 derr) / (n sum|wg|) {float(rel.max()):.2f} x 2^-24, "
                  f"{int(m['reach'].sum())} of {nv * lh * lw} texels reached")
            assert bool((err <= bound).all())
        else:
            untouched = ~m["reach"]
            assert bool(untouched.any()) or lh * lw < 1000           # the small latents are reached everywhere
            assert bool((g_lat[untouched] == start).all())


def logit_regime(kind, R, gen):
    if kind == "uniform":
        return torch.rand(3, R, generator=gen)
    if kind == "spread80":
        return torch.rand(3, R, generator=gen) * 80 - 40
    if kind == "onehot":
        return torch.where(torch.rand(3, R, generator=gen) < 1 / 64, torch.rand(3, R, generator=gen), torch.full((3, R), -1e4))
    if kind == "ties":
        return torch.randint(0, 3, (3, R), generator=gen).float()
    return torch.full((3, R), 0.5)


def softmax_spread(logits, nv):
    """Largest |logit - pillar max| among the cells with a non-zero fp32 softmax weight: the kernel rounds l - max in fp32, an
    absolute error of up to 2^-24 |l - max| in the exponent."""
    lg = logits.double().reshape(3, nv, G, G, G)
    d = torch.stack([lg[a].amax(1 + a, keepdim=True) - lg[a] for a in range(3)])
    return float(d[d < 88].max())


@pytest.mark.parametrize("nv", [1, 3, 8])
@pytest.mark.parametrize("kind", ["uniform", "spread80", "onehot", "ties", "equal"])
def test_pool_matches_model(cuda, nv, kind):
    """Softmax pillar sums and their backward against the model (one view at a time), each upstream plane alone and then all three;
    the backward is bit-identical across two calls.  Bound in units of the magnitudes: (POOL_TOL + POOL_SPREAD_TOL x spread) 2^-24."""
    from neo360_b200 import _lib as L
    R, V = nv * G ** 3, G ** 3
    gen = torch.Generator().manual_seed(11 * nv + len(kind))
    lat = torch.randn(R, 512, generator=gen).to(cuda)
    logits = logit_regime(kind, R, gen).to(cuda)
    spread = softmax_spread(logits, nv)
    tol = (POOL_TOL + POOL_SPREAD_TOL * spread) * U
    out = [torch.empty(nv, 512, G, G, device=cuda) for _ in range(3)]
    L.check(lib().neo_grid_encoder_pool(L.ptr(lat), L.ptr(logits), nv, *[L.ptr(t) for t in out], None))
    ups = {n: torch.randn(nv, 512, G, G, generator=gen).to(cuda) for n in ("xz", "xy", "yz")}
    worst = [0.0, 0.0, 0.0]
    # an element whose products fall in fp32's subnormal range carries an absolute rounding of up to 2^-149 per product and sum
    rel = lambda got, ref, mag: float((((got.double() - ref).abs() - FLOOR) / mag.clamp(min=1e-300)).max())
    for v in range(nv):
        rows = slice(v * V, (v + 1) * V)
        m = etm.pool_fwd(lat[rows], logits[:, rows], 1, G)
        for name, got in zip(("xz", "xy", "yz"), out):
            worst[0] = max(worst[0], rel(got[v:v + 1], m[name], m[name + "_mag"]))
    for sel in (["xz"], ["xy"], ["yz"], ["xz", "xy", "yz"]):
        gs = [ups[n] if n in sel else None for n in ("xz", "xy", "yz")]
        runs = []
        for _ in range(2):
            d_lat, d_lg = torch.empty_like(lat), torch.empty_like(logits)
            L.check(lib().neo_grid_encoder_pool_bwd(L.ptr(lat), L.ptr(logits), nv, *[L.ptr(g) for g in gs], L.ptr(d_lat), L.ptr(d_lg), None))
            runs.append((d_lat, d_lg))
        assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1]), sel
        for v in range(nv):
            rows = slice(v * V, (v + 1) * V)
            mb = etm.pool_bwd(lat[rows], logits[:, rows], 1, G, **{f"g_{n}": ups[n][v:v + 1] for n in sel})
            worst[1] = max(worst[1], rel(runs[0][0][rows], mb["d_lat"], mb["d_lat_mag"]))
            worst[2] = max(worst[2], rel(runs[0][1][:, rows], mb["d_logits"], mb["d_logits_mag"]))
            del mb
        del runs
    w = [x / U for x in worst]
    print(f"pool nv={nv} {kind} (spread {spread:.1f}): fwd max {w[0]:.2f}, bwd d_lat max {w[1]:.2f}, d_logits max {w[2]:.2f} "
          f"x 2^-24 of the magnitudes (bound {tol / U:.1f})")
    assert max(worst) <= tol


def shift_invariant(enc, prefix=""):
    """Biases whose exact gradient is zero: the second aggregator layers' (a softmax does not see a constant shift of its logits) and
    those of the floor-plan convolutions followed by a BatchNorm in train mode.  Both forms return rounding noise for them."""
    names = {f"{prefix}pillar_aggregator_{n}.2.bias" for n in ("xz", "yz", "xy")} | {f"agg_{n}.2.bias" for n in ("xz", "yz", "xy")}
    for pl in ("xy", "yz", "xz"):
        seq = getattr(enc, f"floorplan_convnet_{pl}")
        names |= {f"{prefix}floorplan_convnet_{pl}.{i}.bias" for i in range(len(seq) - 1)
                  if isinstance(seq[i], torch.nn.Conv2d) and isinstance(seq[i + 1], torch.nn.BatchNorm2d)}
    return names


def compare_grads(tag, got, ref, mx=None, l2=None, zero=frozenset()):
    """Per tensor: max error over its largest |reference| and relative L2.  The biases in `zero` (shift_invariant) are held to the
    scale of their weights' gradients instead."""
    worst = (0.0, 0.0)
    mx, l2 = E2E_MAX if mx is None else mx, E2E_L2 if l2 is None else l2
    for name in ref:
        r, g = ref[name].double(), got[name].double().to(ref[name].device)
        if name in zero:
            wscale = float(ref[name[:-len("bias")] + "weight"].double().abs().max())
            assert float((g - r).abs().max()) <= E2E_MAX * wscale, (tag, name)
            continue
        scale = float(r.abs().max())
        if scale == 0:
            assert float(g.abs().max()) == 0, name
            continue
        emax = float((g - r).abs().max()) / scale
        el2 = float(torch.linalg.norm(g - r) / torch.linalg.norm(r))
        worst = (max(worst[0], emax), max(worst[1], el2))
        assert emax <= mx and el2 <= l2, (tag, name, emax, el2)
    print(f"{tag}: {len(ref)} gradients, worst max {worst[0]:.2e} of scale, worst relative L2 {worst[1]:.2e}")


def dense_params(enc):
    mods = {"depth_fc": enc.depth_fc, "agg_xz": enc.pillar_aggregator_xz, "agg_yz": enc.pillar_aggregator_yz, "agg_xy": enc.pillar_aggregator_xy}
    return {f"{k}.{n}": p for k, m in mods.items() for n, p in m.named_parameters()}


def test_end_to_end_matches_float64(cuda):
    """GridEncoder in train mode at NV = 1: the three planes and the gradients of a loss on them with respect to the latent and every
    parameter of depth_fc and the aggregators, CUDA form (fp32) against autograd through the float64 module with dense_torch."""
    from neo360_b200.encoder import GridEncoder
    torch.manual_seed(5)
    enc = GridEncoder().train().to(cuda)
    nv, lh, lw = 1, 60, 80
    W, H = 160, 120
    sc = synth.make_scene((W, H), 3, (4, 4), 1)
    poses, focal, c = sc["src_poses"][:nv].to(cuda), sc["src_focal"][:nv].to(cuda), sc["src_c"][:nv].to(cuda)
    gen = torch.Generator().manual_seed(9)
    latent0 = (torch.rand(nv, 512, lh, lw, generator=gen) ** 2 * 2).to(cuda)
    wts = [torch.randn(nv, 512, G, G, generator=gen).to(cuda) for _ in range(3)]
    latent = latent0.clone().requires_grad_(True)
    planes = enc.dense_train(latent, poses, focal, c, W, H)
    sum(((p * w).sum() for p, w in zip(planes, wts))).backward()
    got = {n: p.grad for n, p in dense_params(enc).items()}
    got["latent"] = latent.grad
    e64 = copy.deepcopy(enc).double()
    lat64 = latent0.double().requires_grad_(True)
    dtype = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        with torch.backends.cudnn.flags(enabled=False):              # float64 grid_sample of 64^3 rows through the native kernel
            ref_planes = e64.dense_torch(lat64, poses.double(), focal.double(), c.double(), W, H)
            sum(((p * w.double()).sum() for p, w in zip(ref_planes, wts))).backward()
    finally:
        torch.set_default_dtype(dtype)
    ref = {n: p.grad for n, p in dense_params(e64).items()}
    ref["latent"] = lat64.grad
    compare_grads("end to end vs float64 dense_torch", got, ref, zero=shift_invariant(enc))
    compare_grads("planes vs float64", {str(i): p.detach() for i, p in enumerate(planes)}, {str(i): p.detach() for i, p in enumerate(ref_planes)})


def encoder_grads(enc, imgs, poses, focal, c, wts):
    enc.zero_grad(set_to_none=True)
    out = enc(imgs, poses, focal, c)
    sum(((o * w).sum() for o, w in zip(out, wts))).backward()
    return {n: p.grad.clone() for n, p in enc.named_parameters() if p.grad is not None}, [o.detach() for o in out]


def test_end_to_end_fp32_production_shape(cuda):
    """NV = 3, 640 x 480 source images (latent 240 x 320): every encoder parameter's gradient and the three outputs of the CUDA form
    against the fp32 dense_torch form on the same GPU."""
    from neo360_b200.encoder import GridEncoder
    torch.manual_seed(6)
    enc = GridEncoder().train().to(cuda)
    sc = synth.make_scene((640, 480), 3, (4, 4), 2)
    poses, focal, c = sc["src_poses"].to(cuda), sc["src_focal"].to(cuda), sc["src_c"].to(cuda)
    gen = torch.Generator().manual_seed(10)
    imgs = (torch.rand(3, 3, 480, 640, generator=gen) * 2 - 1).to(cuda)
    wts = [torch.randn(3, 128, 120, 160, generator=gen).to(cuda) for _ in range(3)]
    got, out = encoder_grads(enc, imgs, poses, focal, c, wts)
    enc.dense_train = enc.dense_torch
    ref, out_ref = encoder_grads(enc, imgs, poses, focal, c, wts)
    assert set(got) == set(ref) and len(ref) == len(list(enc.parameters()))
    compare_grads("fp32 production shape, gradients", got, ref, mx=E2E_FP32_MAX, l2=E2E_FP32_L2, zero=shift_invariant(enc))
    compare_grads("fp32 production shape, outputs", {str(i): o for i, o in enumerate(out)}, {str(i): o for i, o in enumerate(out_ref)})


def test_aggregators_only_receive_gradients(cuda):
    """With only the pillar aggregators trainable, `forward` takes the training path and they receive the framework form's gradients."""
    from neo360_b200.encoder import GridEncoder
    torch.manual_seed(7)
    enc = GridEncoder().train().to(cuda)
    for n, p in enc.named_parameters():
        p.requires_grad_(n.startswith("pillar_aggregator_"))
    sc = synth.make_scene((160, 120), 1, (4, 4), 3)
    gen = torch.Generator().manual_seed(12)
    imgs = (torch.rand(1, 3, 120, 160, generator=gen) * 2 - 1).to(cuda)
    wts = [torch.randn(1, 128, 120, 160, generator=gen).to(cuda) for _ in range(3)]
    args = (imgs, sc["src_poses"].to(cuda), sc["src_focal"].to(cuda), sc["src_c"].to(cuda))
    got, _ = encoder_grads(enc, *args, wts)
    assert sorted(got) == sorted(n for n, p in enc.named_parameters() if p.requires_grad) and len(got) == 12
    enc.dense_train = enc.dense_torch
    ref, _ = encoder_grads(enc, *args, wts)
    compare_grads("aggregators only", got, ref, zero=shift_invariant(enc))


def test_training_step_with_encoder(cuda):
    """One NeO-360 training step, `NeRF_TP(encoder=GridEncoder())` and `training_loss`: every parameter's gradient against the same
    step with `dense_train` patched to `dense_torch` on the encoder instance."""
    from neo360_b200 import NeRF_TP, batches
    from neo360_b200.encoder import GridEncoder
    from neo360_b200.training import training_loss
    torch.manual_seed(0)
    net = NeRF_TP(num_coarse_samples=32, num_fine_samples=16, num_src_views=3, precision="fp32", encoder=GridEncoder())
    sd = net.state_dict()
    sd.update(synth.make_mlp_params(0))
    net.load_state_dict(sd)
    net = net.to(cuda).train()
    sc = synth.make_scene((640, 480), 3, (120, 160), 0)
    g0 = torch.Generator().manual_seed(77)
    src = {"src_poses": sc["src_poses"].to(cuda), "src_focal": sc["src_focal"].to(cuda), "src_c": sc["src_c"].to(cuda),
           "src_imgs": (torch.rand(3, 3, 480, 640, generator=g0) * 2 - 1).to(cuda)}
    g = torch.Generator().manual_seed(1234)
    tposes = torch.stack([synth.target_pose(5 * k, 100)[:3, :4] for k in range(batches.NUM_TARGET_VIEWS)]).to(cuda)
    views = batches.TargetViews(tposes, torch.rand(batches.NUM_TARGET_VIEWS, 480, 640, 3, generator=g).to(cuda), 0.8 * 640)
    pix = batches.draw_pix_inds(views.T, views.H, views.W, 512, g)
    batch = batches.train_batch(views, src, pix_inds=pix)

    def step():
        net.zero_grad(set_to_none=True)
        torch.manual_seed(1)
        ret = net(batch, True, False, None, None, out_depth=False)
        training_loss(ret, batch["target"]).backward()
        return {n: p.grad.clone() for n, p in net.named_parameters() if p.grad is not None}

    got = step()
    net.encoder.dense_train = net.encoder.dense_torch
    ref = step()
    assert set(got) == set(ref) and any(n.startswith("encoder.depth_fc") for n in ref)
    compare_grads("training step with the encoder", got, ref, zero=shift_invariant(net.encoder, "encoder."))
