"""CPU: the float64 model of the GridEncoder training stages (oracle/encoder_train_model.py) against autograd through
`GridEncoder.dense_torch`, and the argument checks of the four training entry points (no GPU needed)."""
import pytest
import torch

from neo360_b200 import synth
from oracle import encoder_train_model as etm

G = 8


def small_encoder():
    from neo360_b200.encoder import GridEncoder
    torch.manual_seed(3)
    enc = GridEncoder().double()
    enc.GRID = G
    return enc


def encoder_poses(nv):
    """Synthetic source cameras plus an identity camera (grid cells on z_cam = 0 and behind the camera) and one at (0, 0, 0.5)."""
    poses = synth.make_scene((36, 22), nv, (4, 4), 0)["src_poses"].double()
    poses[0] = torch.eye(4, dtype=torch.float64)
    if nv > 1:
        poses[1] = torch.eye(4, dtype=torch.float64)
        poses[1, 2, 3] = 0.5
    return poses


def md(a, b):
    return float((a.detach() - b.detach()).abs().max())


@pytest.mark.parametrize("nv,lat_hw", [(1, (11, 18)), (3, (19, 12))])
def test_model_without_rounding_is_dense_torch_autograd(nv, lat_hw):
    """G = 8, float64 (the default dtype too, as dense_torch builds its grid in it): the features, the pool forward, the pool backward
    (each upstream plane alone and all three together) and the latent gradient of the model equal autograd through dense_torch."""
    enc = small_encoder()
    lh, lw = lat_hw
    W, H = 2 * lw, 2 * lh
    latent = (torch.rand(nv, 512, lh, lw, generator=torch.Generator().manual_seed(nv), dtype=torch.float64) ** 2 * 2).requires_grad_(True)
    poses = encoder_poses(nv)
    focal, c = torch.full((nv,), 0.8 * W, dtype=torch.float64), torch.tensor([[W / 2.0, H / 2.0]] * nv, dtype=torch.float64)
    cap = {}
    hooks = [enc.depth_fc.register_forward_hook(lambda m, i, o: cap.update(X=i[0], lat=o))]
    for n in etm.AXES:
        hooks.append(getattr(enc, f"pillar_aggregator_{n}").register_forward_hook(lambda m, i, o, n=n: cap.update({n: o})))
    dtype = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        planes = dict(zip(("xz", "xy", "yz"), enc.dense_torch(latent, poses, focal, c, W, H)))
        tp, cam, dvec = etm.features_taps(G, (lh, lw), poses, float(focal[0]), c[0], W, H, fp32=False)
        R = nv * G ** 3
        # features
        X = etm.features_fwd(latent.detach(), tp, cam, dvec)["X"]
        Xr = cap["X"].reshape(R, 518)
        assert md(X, Xr) <= 1e-12 * float(Xr.detach().abs().max())
        # pool forward at dense_torch's own rows and logits
        lat = cap["lat"].reshape(R, 512)
        logits = torch.stack([cap[n].reshape(R) for n in etm.AXES])
        pf = etm.pool_fwd(lat.detach(), logits.detach(), nv, G)
        for n in ("xz", "xy", "yz"):
            assert md(pf[n], planes[n]) <= 1e-12 * float(planes[n].detach().abs().max()), n
        # pool backward: each upstream plane alone, then all three
        gen = torch.Generator().manual_seed(7 + nv)
        ups = {n: torch.randn(planes[n].shape, generator=gen, dtype=torch.float64) for n in planes}
        for sel in (["xz"], ["xy"], ["yz"], ["xz", "xy", "yz"]):
            outs, gs = [planes[n] for n in sel], [ups[n] for n in sel]
            refs = torch.autograd.grad(outs, [cap["lat"]] + [cap[n] for n in etm.AXES], gs, retain_graph=True, allow_unused=True,
                                       materialize_grads=True)
            pb = etm.pool_bwd(lat.detach(), logits.detach(), nv, G, **{f"g_{n}": ups[n] for n in sel})
            for a, n in enumerate(etm.AXES):
                ref = refs[1 + a].reshape(R)
                assert md(pb["d_logits"][a], ref) <= 1e-12 * (1 + float(ref.abs().max())), (sel, n)
                assert bool((pb["d_logits_mag"][a] >= pb["d_logits"][a].abs() - 1e-12).all())
            # the direct path of lat plus its path through the aggregators = autograd's gradient of lat
            via_agg = torch.autograd.grad([cap[n] for n in etm.AXES], cap["lat"], [pb["d_logits"][a].reshape(cap[n].shape)
                                                                                  for a, n in enumerate(etm.AXES)], retain_graph=True)[0]
            ref = refs[0].reshape(R, 512)
            assert md(pb["d_lat"] + via_agg.reshape(R, 512), ref) <= 1e-12 * float(ref.abs().max()), sel
        # latent gradient through the lookup adjoint
        gs = [ups[n] for n in ("xz", "xy", "yz")]
        g_X, g_lat = torch.autograd.grad([planes[n] for n in ("xz", "xy", "yz")], [cap["X"], latent], gs)
        fb = etm.features_bwd(tp, g_X.reshape(R, 518), nv)
        ref = g_lat.permute(0, 2, 3, 1)
        assert float(ref.abs().max()) > 0
        assert md(fb["val"], ref) <= 1e-12 * float(ref.abs().max())
    finally:
        torch.set_default_dtype(dtype)
        for h in hooks:
            h.remove()
    # the scene exercises cells behind the camera, on z_cam = 0, and lookups outside the latent
    assert bool((cam[:, 2] >= 1e-3).any()) and bool((cam[:, 2] == 0).any()) and bool((tp["w"] == 0).all(-1).any())


@pytest.fixture(scope="module")
def lib():
    from neo360_b200 import build, _lib
    build.build()
    return _lib.load()


def test_training_entry_points_reject_bad_arguments_without_gpu(lib):
    """The four training entry points reject NULL buffers, nv < 1, latent sizes < 2, image sizes <= 0, strides and alignments their
    kernels cannot address -- all before any launch (the data pointers are never dereferenced)."""
    p = 1 << 20
    feat = lambda lat=p, nv=1, lh=4, lw=4, w=8, h=8, poses=p, X=p, ldx=520: lib.neo_grid_encoder_features(lat, nv, lh, lw, w, h, poses, 1.0,
                                                                                                       0.0, 0.0, X, ldx, None)
    for kw in (dict(lat=None), dict(poses=None), dict(X=None), dict(nv=0), dict(lh=1), dict(lw=1), dict(w=0), dict(h=-1), dict(ldx=516),
               dict(ldx=518), dict(ldx=644), dict(lat=p + 4), dict(X=p + 8)):
        assert feat(**kw) == -1, kw
    assert b"neo_grid_encoder_features" in lib.neo_last_error()
    bwd = lambda nv=1, lh=4, lw=4, w=8, h=8, poses=p, g=p, ldg=518, gl=p: lib.neo_grid_encoder_features_bwd(nv, lh, lw, w, h, poses, 1.0, 0.0,
                                                                                                         0.0, g, ldg, gl, None)
    for kw in (dict(poses=None), dict(g=None), dict(gl=None), dict(nv=0), dict(lh=1), dict(w=0), dict(ldg=510), dict(ldg=519),
               dict(g=p + 4), dict(gl=p + 8)):
        assert bwd(**kw) == -1, kw
    assert b"neo_grid_encoder_features_bwd" in lib.neo_last_error()
    pool = lambda lat=p, lg=p, nv=1, o=(p, p, p): lib.neo_grid_encoder_pool(lat, lg, nv, *o, None)
    for kw in (dict(lat=None), dict(lg=None), dict(nv=0), dict(o=(p, None, p)), dict(lat=p + 4)):
        assert pool(**kw) == -1, kw
    assert b"neo_grid_encoder_pool" in lib.neo_last_error()
    pb = lambda lat=p, lg=p, nv=1, dl=p, dg=p: lib.neo_grid_encoder_pool_bwd(lat, lg, nv, None, None, None, dl, dg, None)
    for kw in (dict(lat=None), dict(lg=None), dict(nv=0), dict(dl=None), dict(dg=None)):
        assert pb(**kw) == -1, kw
    assert b"neo_grid_encoder_pool_bwd" in lib.neo_last_error()
