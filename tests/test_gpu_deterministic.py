"""GPU: training under torch.use_deterministic_algorithms(True).

* lookups: `neo_index_maps_bwd_det` (and the raw-map calls `_Lookup` makes with it) and `neo_grid_encoder_features_bwd_det` equal the fp32
  emulation of their segmented reduction over their own workspace entries bit for bit (oracle/det_model.segment_emulate), stay within the
  float64 bounds the atomic path is held to (tests/test_gpu_train_stages.check_scatter, the encoder's FEAT_BWD_TOL), leave texels no
  entry reaches at their sentinel, and two calls are bit-identical.
* losses: `neo_distortion_loss(_bwd)` and `neo_interlevel_loss(_bwd)` per ray within the a-priori bounds of oracle/det_model.py, two calls
  bit-identical; N = 1, all-zero weights, opaque rays, descending (bg) m.
* upsampling: `neo_upsample_bilinear_bwd` within its bound of the float64 adjoint at every shape the encoder uses.
* end to end, in a subprocess that sets CUBLAS_WORKSPACE_CONFIG before CUDA starts: three Adam steps from one seed, twice, for NeO-360 with
  GridEncoder in the step (projected and reference formulation), NeO-360 with a frozen encoder, vanilla NeRF and Mip-NeRF 360: every loss,
  parameter and Adam state bit-identical between the runs; one deterministic step's gradients against the default path's.
"""
import gc
import json
import os
import subprocess
import sys

import pytest
import torch

from oracle import det_model as dm
from oracle import encoder_train_model as etm
from test_gpu_encoder_train import FEAT_BWD_TOL, G, geometry, ill_rows
from test_gpu_train_stages import Geo, check_scatter, contention_points, level1_points, sentinel, split_near, training_poses

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PLANE_HW, LAT_HW, IMG_WH = (120, 160), (240, 320), (640, 480)


@pytest.fixture(scope="module")
def cuda():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from neo360_b200 import build
    build.build()
    return torch.device("cuda:0")


def free_device_memory():
    """Return what this process keeps cached on the device (the framework's caching allocator and the library's pool of scene blocks)."""
    import neo360_b200
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    neo360_b200.release_cached()


@pytest.fixture(autouse=True)
def release_memory():
    """The production-shape cases cache tens of GB; the end-to-end case runs in a subprocess that needs that memory back."""
    yield
    free_device_memory()


def L():
    from neo360_b200 import _lib
    return _lib


def stream():
    return torch.cuda.current_stream().cuda_stream


def maps_bwd_det(geo, pts, C, gl, gw, glat, gpl):
    lib = L().load()
    M = pts.shape[0]
    need = lib.neo_index_maps_bwd_det_workspace_bytes(geo.h, M, C)
    assert need > 0
    ws = torch.empty(need, dtype=torch.uint8, device=pts.device)
    P = L().ptr
    L().check(lib.neo_index_maps_bwd_det(geo.h, P(pts), M, C, P(gl), P(gw), P(glat), *(P(x) for x in (gpl or [None] * 3)), P(ws), need,
                                         stream()))
    assert lib.neo_index_maps_bwd_det(geo.h, P(pts), M, C, P(gl), P(gw), P(glat), *(P(x) for x in (gpl or [None] * 3)), P(ws), need - 1,
                                      stream()) == -1                                 # a short workspace is refused before any launch
    return ws


def run_lookup_case(label, geo, pts, C, dev, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    nv, (Hp, Wp), (Hl, Wl) = geo.nv, geo.plane_hw, geo.lat_hw
    reg, _ = split_near(geo, pts)
    M = reg.shape[0]
    gl = torch.randn(nv * M, C, generator=g, device=dev)
    gw = torch.randn(nv * M, C, generator=g, device=dev)
    outs = []
    for _ in range(2):
        glat = sentinel((nv, Hl, Wl, C), dev)
        gpl = [sentinel((nv, Hp, Wp, C), dev) for _ in range(3)]
        ws = maps_bwd_det(geo, reg, C, gl, gw, glat, gpl)
        outs.append((glat, gpl, ws))
    (glat, gpl, ws), (glat2, gpl2, _) = outs
    assert torch.equal(glat, glat2) and all(torch.equal(a, b) for a, b in zip(gpl, gpl2)), f"{label}: two calls differ"
    rows = nv * M
    E, T_lat, hw = 16 * rows, nv * Hl * Wl, nv * Hp * Wp
    T = T_lat + 3 * hw
    ks, ids, wts = dm.read_entries(ws, E, T)
    g_of = lambda e: torch.where((e < 4 * rows)[:, None], gl[(e // 4).clamp(max=rows - 1)], gw[((e - 4 * rows).clamp(min=0) // 12)])
    init = torch.cat([sentinel((nv, Hl, Wl, C), dev).reshape(-1, C)] + [sentinel((nv, Hp, Wp, C), dev).reshape(-1, C)] * 3)
    emu = dm.segment_emulate(ks, ids, wts, g_of, init)
    got = torch.cat([glat.reshape(-1, C)] + [x.reshape(-1, C) for x in gpl])
    assert torch.equal(got, emu), f"{label}: kernel differs from the fp32 emulation of its own entries"
    tw, tl = geo.taps(reg, False), geo.taps(reg, True)
    sent_l, sent_p = sentinel((nv, Hl, Wl, C), dev), sentinel((nv, Hp, Wp, C), dev)
    check_scatter(f"{label} det local", glat, sent_l, tl[0], gl, nv, 1 << 26)
    for name, tp, x in zip(("xz", "xy", "yz"), tw, gpl):
        check_scatter(f"{label} det {name}", x, sent_p, tp, gw, nv, 1 << 26)


@pytest.mark.parametrize("nv", [1, 3, 8])
def test_index_maps_bwd_det(cuda, nv):
    geo = Geo(training_poses(nv), PLANE_HW, LAT_HW, IMG_WH, cuda)
    for C in (4, 128, 260, 512):
        run_lookup_case(f"nv={nv} C={C} batch 512 rays", geo, level1_points(512, 31, cuda), C, cuda, C + nv)
    run_lookup_case(f"nv={nv} C=128 contention", geo, contention_points(cuda), 128, cuda, 5)


def test_index_maps_bwd_det_production_shape(cuda):
    """The lookup calls of a 4096-ray step: nv 3, the projected maps' 256 channels."""
    geo = Geo(training_poses(3), PLANE_HW, LAT_HW, IMG_WH, cuda)
    run_lookup_case("nv=3 C=256 4096 rays", geo, level1_points(4096, 37, cuda), 256, cuda, 7)


def test_lookup_wrappers_use_det_in_deterministic_mode(cuda):
    """_Lookup (two det calls, C 128 / 512) and _LookupMaps record the mode in forward: bit-identical gradients across two backward passes."""
    from neo360_b200.training import _Lookup, _LookupMaps
    nv = 3
    g = torch.Generator(device=cuda).manual_seed(41)
    (Hp, Wp), (Hl, Wl) = PLANE_HW, LAT_HW
    raw = [torch.randn(nv, 128, Hp, Wp, generator=g, device=cuda) for _ in range(3)] + [torch.randn(nv, 512, Hl, Wl, generator=g, device=cuda)]
    geo = Geo(training_poses(nv), PLANE_HW, LAT_HW, IMG_WH, cuda, raw=raw)
    reg, _ = split_near(geo, level1_points(64, 43, cuda))
    C = 256                                             # _LookupMaps takes four maps of one channel count (the projected maps)
    proj = [torch.randn(nv, Hl, Wl, C, generator=g, device=cuda)] + [torch.randn(nv, Hp, Wp, C, generator=g, device=cuda) for _ in range(3)]
    grads = []
    torch.use_deterministic_algorithms(True)
    try:
        for _ in range(2):
            leaves = [x.clone().requires_grad_(True) for x in raw + proj]
            world, local = _Lookup.apply(reg, *leaves[:4], geo.net)
            lp, wp = _LookupMaps.apply(reg, *leaves[4:], geo.net)
            gg = torch.Generator(device=cuda).manual_seed(1)
            loss = sum((t * torch.randn(t.shape, generator=gg, device=cuda)).sum() for t in (world, local, lp, wp))
            loss.backward()
            grads.append([x.grad.clone() for x in leaves])
    finally:
        torch.use_deterministic_algorithms(False)
    assert all(torch.equal(a, b) for a, b in zip(*grads))


@pytest.mark.parametrize("nv,lat_hw", [(1, (11, 18)), (3, (19, 12)), (8, (11, 18)), (3, (240, 320))])
def test_features_bwd_det(cuda, nv, lat_hw):
    lib = L().load()
    P = L().ptr
    poses, focal, c, W, H = geometry(nv, lat_hw)
    lh, lw = lat_hw
    R = nv * G ** 3
    gen = torch.Generator().manual_seed(nv + lh)
    pc = poses.float().contiguous().to(cuda)
    geo = (nv, lh, lw, W, H)
    cam_args = (float(focal[0]), float(c[0, 0]), float(c[0, 1]))
    tp, _, _ = etm.features_taps(G, lat_hw, poses.to(cuda), float(focal[0]), c[0], W, H)
    ill = ill_rows(nv, lat_hw, poses, focal, c, W, H, cuda)
    g = torch.randn(R, 518, generator=gen).to(cuda)
    g[ill] = 0
    need = lib.neo_grid_encoder_features_bwd_det_workspace_bytes(nv, lh, lw)
    assert need > 0
    outs = []
    for _ in range(2):
        ws = torch.empty(need, dtype=torch.uint8, device=cuda)
        g_lat = torch.full((nv, lh, lw, 512), -3.0, device=cuda)
        L().check(lib.neo_grid_encoder_features_bwd_det(*geo, P(pc), *cam_args, P(g), 518, P(g_lat), P(ws), need, None))
        outs.append((g_lat, ws))
    assert torch.equal(outs[0][0], outs[1][0])
    g_lat, ws = outs[0]
    E, T = 4 * R, nv * lh * lw
    ks, ids, wts = dm.read_entries(ws, E, T)
    emu = dm.segment_emulate(ks, ids, wts, lambda e: g[e // 4, :512], torch.full((T, 512), -3.0, device=cuda))
    assert torch.equal(g_lat.reshape(T, 512), emu)
    m = etm.features_bwd(tp, g, nv)
    err = (g_lat.double() + 3.0 - m["val"]).abs()
    n = m["n"][..., None].clamp(min=1)
    assert bool((err <= FEAT_BWD_TOL * n * (m["mag"] + 3.0) + 2 * m["derr"]).all())
    assert bool((g_lat[~m["reach"]] == -3.0).all())


def loss_inputs(n, N, seed, dev, descending=False):
    g = torch.Generator().manual_seed(seed)
    w = torch.rand(n, N, generator=g) ** 3
    w[0] = 0                                                              # all-zero weights
    if N > 1:
        w[1] = 0
        w[1, N // 2] = 1.0                                                # an opaque ray
    m = torch.sort(torch.rand(n, N, generator=g), -1, descending=descending).values
    I = torch.rand(n, N, generator=g) / N
    return w.to(dev), m.to(dev), I.to(dev), torch.randn(n, generator=g).to(dev)


@pytest.mark.parametrize("descending", [False, True], ids=["fg", "bg descending m"])
@pytest.mark.parametrize("N", [1, 31, 32, 33, 129, 193])
def test_distortion_kernels(cuda, N, descending):
    lib, P = L().load(), L().ptr
    n = 4096
    w, m, I, g = loss_inputs(n, N, N, cuda, descending)
    res = []
    for _ in range(2):
        out, dw = torch.empty(n, device=cuda), torch.empty(n, N, device=cuda)
        L().check(lib.neo_distortion_loss(P(w), P(m), P(I), 0.0, n, N, P(out), stream()))
        L().check(lib.neo_distortion_loss_bwd(P(w), P(m), P(I), 0.0, n, N, P(g), P(dw), stream()))
        res.append((out, dw))
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1])
    out, dw = res[0]
    lb, gb = dm.distortion_bounds(w, m, I, g)
    r1 = float(((out.double() - dm.distortion64(w, m, I)).abs() / lb.clamp_min(1e-300)).max())
    r2 = float(((dw.double() - dm.distortion_grad64(w, m, I, g)).abs() / gb.clamp_min(1e-300)).max())
    print(f"distortion N={N} {'desc' if descending else 'asc'}: loss {r1:.3g}, grad {r2:.3g} of the bound")
    assert r1 <= 1 and r2 <= 1
    out2 = torch.empty(n, device=cuda)                                  # a scalar interval is the same as a constant tensor
    L().check(lib.neo_distortion_loss(P(w), P(m), None, 0.25, n, N, P(out2), stream()))
    L().check(lib.neo_distortion_loss(P(w), P(m), P(torch.full_like(w, 0.25)), 0.0, n, N, P(out), stream()))
    assert torch.equal(out, out2)


@pytest.mark.parametrize("Nc,Np", [(1, 1), (32, 64), (64, 64), (8, 160)])
def test_interlevel_kernels(cuda, Nc, Np):
    lib, P = L().load(), L().ptr
    n = 2048
    gen = torch.Generator().manual_seed(Nc * Np)
    c = torch.sort(torch.rand(n, Nc + 1, generator=gen), -1).values
    te = torch.sort(torch.rand(n, Np + 1, generator=gen), -1).values
    if Np >= 6:
        te[:, 3:6] = te[:, 3:4]
        c[:, 1] = te[:, 3]
        c = torch.sort(c, -1).values
    w = torch.rand(n, Nc, generator=gen) ** 2
    we = torch.rand(n, Np, generator=gen) ** 2
    w[0], we[1] = 0, 0
    g = torch.randn(n, generator=gen)
    c, te, w, we, g = (x.to(cuda) for x in (c, te, w, we, g))
    res = []
    for _ in range(2):
        out, dwe = torch.empty(n, device=cuda), torch.empty(n, Np, device=cuda)
        L().check(lib.neo_interlevel_loss(P(c), P(w), P(te), P(we), n, Nc, Np, P(out), stream()))
        L().check(lib.neo_interlevel_loss_bwd(P(c), P(w), P(te), P(we), n, Nc, Np, P(g), P(dwe), stream()))
        res.append((out, dwe))
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1])
    out, dwe = res[0]
    lb, gb = dm.interlevel_bounds(c, w, te, we, g)
    r1 = float(((out.double() - dm.interlevel64(c, w, te, we)).abs() / lb.clamp_min(1e-300)).max())
    r2 = float(((dwe.double() - dm.interlevel_grad64(c, w, te, we, g)).abs() / gb.clamp_min(1e-300)).max())
    print(f"interlevel {Nc}/{Np}: loss {r1:.3g}, grad {r2:.3g} of the bound")
    assert r1 <= 1 and r2 <= 1


# SpatialEncoder at 640 x 480 (feats at 1/2, 1/4, 1/8, 1/16 -> 240 x 320, the first an identity) and the floor-plan stacks (16 -> 32,
# 32 -> 120 x 160); smaller images for the other sizes
UP_SHAPES = [((240, 320), (240, 320)), ((120, 160), (240, 320)), ((60, 80), (240, 320)), ((30, 40), (240, 320)), ((16, 16), (32, 32)),
             ((32, 32), (120, 160)), ((60, 80), (120, 160)), ((1, 1), (4, 4)), ((5, 3), (1, 1))]


@pytest.mark.parametrize("hw_in,hw_out", UP_SHAPES)
def test_upsample_bwd(cuda, hw_in, hw_out):
    lib, P = L().load(), L().ptr
    planes = 6
    gy = torch.randn(planes, *hw_out, generator=torch.Generator().manual_seed(3)).to(cuda)
    res = []
    for _ in range(2):
        gx = torch.empty(planes, *hw_in, device=cuda)
        L().check(lib.neo_upsample_bilinear_bwd(P(gy), planes, *hw_in, *hw_out, P(gx), stream()))
        res.append(gx)
    assert torch.equal(res[0], res[1])
    ratio = float(((res[0].double() - dm.upsample_adjoint64(gy, hw_in)).abs() / dm.upsample_bound(gy, hw_in).clamp_min(1e-300)).max())
    print(f"upsample {hw_in} -> {hw_out}: {ratio:.3g} of the bound")
    assert ratio <= 1
    if hw_in == hw_out:
        assert torch.equal(res[0], gy)


WORKER = r"""
import json, os, sys
os.environ["CUBLAS_WORKSPACE_CONFIG"] = ":4096:8"
sys.path.insert(0, sys.argv[1])
import torch
torch.use_deterministic_algorithms(True)
torch.backends.cudnn.benchmark = False
torch.backends.cuda.matmul.allow_tf32 = False
torch.backends.cudnn.allow_tf32 = False
from neo360_b200 import synth, batches, training, mip
from oracle import neo360_oracle as orc
dev = torch.device("cuda:0")


def neo(case):
    from neo360_b200 import NeRF_TP
    from neo360_b200.encoder import GridEncoder
    W, H = 320, 240
    enc = GridEncoder() if case != "neo frozen encoder" else None
    net = NeRF_TP(num_coarse_samples=32, num_fine_samples=16, num_src_views=3, precision="fp32", encoder=enc)
    sd = net.state_dict()
    sd.update(synth.make_mlp_params(0))
    net.load_state_dict(sd)
    net = net.to(dev).train()
    net.train_projected = case != "neo encoder reference"
    sc = synth.make_scene((W, H), 3, (120, 160), 0)
    src = {k: sc[k].to(dev) for k in ("src_poses", "src_focal", "src_c")}
    leaves = {}
    if enc is not None:
        src["src_imgs"] = (torch.rand(3, 3, H, W, generator=torch.Generator().manual_seed(77)) * 2 - 1).to(dev)
        params = [p for p in net.parameters() if p.requires_grad]
    else:
        src["src_imgs"] = torch.empty(3, 3, H, W, device="meta")
        leaves = {k: sc[k].to(dev).requires_grad_(True) for k in ("planes_xz", "planes_xy", "planes_yz", "latent")}
        params = [p for m in net._mlps() for p in m.parameters()] + list(leaves.values())
    g = torch.Generator().manual_seed(1234)
    tposes = torch.stack([synth.target_pose(5 * k, 100)[:3, :4] for k in range(batches.NUM_TARGET_VIEWS)]).to(dev)
    views = batches.TargetViews(tposes, torch.rand(batches.NUM_TARGET_VIEWS, H, W, 3, generator=g).to(dev), 0.8 * W)

    def loss_fn(step):
        pix = batches.draw_pix_inds(views.T, views.H, views.W, 256, torch.Generator().manual_seed(step))
        batch = batches.train_batch(views, src, pix_inds=pix)
        batch.update(leaves)
        ret = net(batch, True, False, None, None, out_depth=False)
        return training.training_loss(ret, batch["target"])
    return params, loss_fn


def vanilla(case):
    from neo360_b200.vanilla import NeRF
    net = NeRF(num_coarse_samples=64, num_fine_samples=64)
    net.load_state_dict(synth.make_vanilla_params(0))
    net = net.to(dev).train()
    ro, vd, rd, _ = orc.rays_from_pose(orc.ray_directions(24, 32, 0.8 * 32), synth.target_pose(5, 100)[:3, :4])
    rays = {"rays_o": ro[:256].to(dev), "rays_d": rd[:256].to(dev), "viewdirs": vd[:256].to(dev)}
    tgt = torch.rand(256, 3, generator=torch.Generator().manual_seed(9)).to(dev)

    def loss_fn(step):
        ret = net(rays, True, False, 2.0, 6.0)
        return ((ret[0][0] - tgt) ** 2).mean() + ((ret[1][0] - tgt) ** 2).mean()
    return list(net.parameters()), loss_fn


def mipnerf(case):
    from neo360_b200.mip import MipNeRF360
    net = MipNeRF360(num_prop_samples=64, num_nerf_samples=32)
    net.load_state_dict(synth.make_mip_params(0))
    net = net.to(dev).train()
    ro, vd, rd, radii = orc.rays_from_pose(orc.ray_directions(48, 64, 0.8 * 64), synth.target_pose(9, 100)[:3, :4])
    rays = {"rays_o": ro[:256].to(dev), "rays_d": rd[:256].to(dev), "viewdirs": vd[:256].to(dev), "radii": radii[:256].reshape(-1, 1).to(dev)}
    tgt = torch.rand(256, 3, generator=torch.Generator().manual_seed(9)).to(dev)

    def loss_fn(step):
        ren, hist = net(rays, 0.5, True, True, 0.2, 6.0)
        return mip.training_loss(ren, hist, tgt)
    return [p for p in net.parameters() if p.requires_grad], loss_fn


def run(case, make):
    torch.manual_seed(0)
    params, loss_fn = make(case)
    opt = torch.optim.Adam(params, lr=5e-4)
    losses = []
    for step in range(3):
        torch.manual_seed(100 + step)
        loss = loss_fn(step)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
        losses.append(loss.detach().clone())
    state = [t.detach().clone() for p in params for t in [p] + [v for v in opt.state[p].values() if torch.is_tensor(v)]]
    return losses, state


def grads(make, case, det):
    torch.use_deterministic_algorithms(det)
    torch.manual_seed(0)
    params, loss_fn = make(case)
    torch.manual_seed(100)
    loss_fn(0).backward()
    out = [p.grad.detach().clone() for p in params]
    torch.use_deterministic_algorithms(True)
    return out


out = {}
cases = [("neo encoder projected", neo), ("neo encoder reference", neo), ("neo frozen encoder", neo), ("vanilla configs[0]", vanilla),
         ("mip 64/64/32", mipnerf)]
import gc
for case, make in cases:
    try:
        a, b = run(case, make), run(case, make)
        same = all(torch.equal(x, y) for x, y in zip(a[0] + a[1], b[0] + b[1]))
        out[case] = {"identical": same, "losses": [float(x) for x in a[0]]}
    except Exception as e:
        out[case] = {"error": f"{type(e).__name__}: {e}"}
    a = b = None
    gc.collect()
    torch.cuda.empty_cache()
for case, make in (("neo frozen encoder", neo), ("mip 64/64/32", mipnerf)):
    try:
        gd, gn = grads(make, case, True), grads(make, case, False)
        worst = max(float((x - y).abs().max()) / max(float(y.abs().max()), 1e-12) for x, y in zip(gd, gn))
        worst2 = max(float((x - y).norm()) / max(float(y.norm()), 1e-30) for x, y in zip(gd, gn))
        out[case + " vs default"] = {"max_rel": worst, "l2_rel": worst2}
    except Exception as e:
        out[case + " vs default"] = {"error": f"{type(e).__name__}: {e}"}
print("RESULT " + json.dumps(out))
"""


def test_training_steps_reproducible_in_deterministic_mode(cuda):
    """Three Adam steps, twice, per model: bit-identical losses, parameters and Adam state; deterministic gradients within the default
    path's bounds (tests/test_training.py: 1e-2 of the gradient scale in max norm, 3e-3 relative L2)."""
    free_device_memory()
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    res = subprocess.run([sys.executable, "-c", WORKER, ROOT], capture_output=True, text=True, env=env, timeout=3000)
    line = [ln for ln in res.stdout.splitlines() if ln.startswith("RESULT ")]
    assert line, res.stdout[-3000:] + res.stderr[-3000:]
    out = json.loads(line[0][len("RESULT "):])
    for case, r in out.items():
        print(case, r)
    for case, r in out.items():
        assert "error" not in r, (case, r)
        if "identical" in r:
            assert r["identical"], case
        else:
            assert r["max_rel"] < 1e-2 and r["l2_rel"] < 3e-3, (case, r)
