"""CPU: the float64 model of GridEncoder's tensor-core training form (oracle/encoder_train_tc_model.py) against autograd through
`GridEncoder.dense_torch`, the stacked first layer of the aggregators against the three separate layers, and the argument checks of its
entry points (no GPU needed)."""
import pytest
import torch

from oracle import encoder_train_tc_model as tcm
from test_encoder_train_model import G, encoder_poses, small_encoder


def grads_by_model_name(enc):
    """nn.Linear parameters of depth_fc and the aggregators under the model's gradient names."""
    fc = enc.depth_fc
    out = {}
    for i, m in enumerate((fc.common_branch[0], fc.common_branch[2], fc.depth_encoder)):
        out[f"w{i}"], out[f"b{i}"] = m.weight, m.bias
    for n in tcm.AXES:
        agg = getattr(enc, f"pillar_aggregator_{n}")
        out[f"{n}_w0"], out[f"{n}_b0"], out[f"{n}_w1"], out[f"{n}_b1"] = agg[0].weight, agg[0].bias, agg[2].weight, agg[2].bias
    return out


@pytest.mark.parametrize("nv,lat_hw", [(1, (11, 18)), (3, (19, 12))])
def test_model_without_rounding_is_dense_torch_autograd(nv, lat_hw):
    """G = 8, float64: with every bf() off, the model's floor plans, logits, latent-row gradient and every parameter gradient of depth_fc
    and the aggregators equal autograd through dense_torch."""
    enc = small_encoder()
    lh, lw = lat_hw
    W, H = 2 * lw, 2 * lh
    latent = (torch.rand(nv, 512, lh, lw, generator=torch.Generator().manual_seed(nv), dtype=torch.float64) ** 2 * 2).requires_grad_(True)
    poses = encoder_poses(nv)
    focal, c = torch.full((nv,), 0.8 * W, dtype=torch.float64), torch.tensor([[W / 2.0, H / 2.0]] * nv, dtype=torch.float64)
    cap = {}
    hooks = [enc.depth_fc.register_forward_hook(lambda m, i, o: cap.update(X=i[0]))]
    for n in tcm.AXES:
        hooks.append(getattr(enc, f"pillar_aggregator_{n}").register_forward_hook(lambda m, i, o, n=n: cap.update({n: o})))
    dtype = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        planes = dict(zip(("xz", "xy", "yz"), enc.dense_torch(latent, poses, focal, c, W, H)))
        R = nv * G ** 3
        X = cap["X"].reshape(R, 518)
        got, logits, S = tcm.forward(X.detach(), tcm.grid_coords(G, nv, torch.float64), tcm.params_of(enc), nv, G, rnd=False)
        for n in planes:
            ref = planes[n].detach()
            assert float((got[n] - ref).abs().max()) <= 1e-12 * float(ref.abs().max()), n
        ref_lg = torch.stack([cap[n].reshape(R) for n in tcm.AXES]).detach()
        assert float((logits - ref_lg).abs().max()) <= 1e-12 * float(ref_lg.abs().max())
        gen = torch.Generator().manual_seed(5 + nv)
        ups = {n: torch.randn(planes[n].shape, generator=gen, dtype=torch.float64) for n in planes}
        P = grads_by_model_name(enc)
        names = list(P)
        refs = torch.autograd.grad([planes[n] for n in ups], [P[k] for k in names] + [cap["X"]], [ups[n] for n in ups])
        mb = tcm.backward(ups["xz"], ups["xy"], ups["yz"], S, tcm.params_of(enc), nv, G, rnd=False)
        grads = dict(zip(names + ["g_X"], refs))
        for k, ref in grads.items():
            ref = ref.reshape(R, 518)[:, :512] if k == "g_X" else ref
            assert mb[k].shape == ref.shape, k
            if k.endswith("_b1"):       # exactly zero (a softmax does not see a shift of its logits): both are rounding noise
                assert float((mb[k] - ref).abs().max()) <= 1e-11 * float(grads[k[:-2] + "w1"].abs().max()), k
                continue
            assert float(ref.abs().max()) > 0, k
            assert float((mb[k] - ref).abs().max()) <= 1e-11 * float(ref.abs().max()), k
    finally:
        torch.set_default_dtype(dtype)
        for h in hooks:
            h.remove()


def test_stacked_first_layer_equals_three_aggregators():
    """The stacked weight U holds each aggregator's 513 columns and zeros elsewhere, so [lat | x y z | 0] U^T + c is, block by block,
    each aggregator's own first layer on [lat | its coordinate].  Integer-valued operands make every product and sum exact in float64,
    so the two forms are compared bit for bit whatever order the matrix products sum in."""
    gen = torch.Generator().manual_seed(2)
    R = 3 * G ** 3
    lat = torch.randint(-8, 9, (R, 512), generator=gen).double()
    coords = torch.randint(-4, 5, (R, 3), generator=gen).double()
    u = [torch.randint(-8, 9, (512, 513), generator=gen).double() for _ in range(3)]
    c = [torch.randint(-8, 9, (512,), generator=gen).double() for _ in range(3)]
    U = tcm.stack_first_layers(u)
    assert U.shape == (1536, 576)
    Lb = torch.cat([lat, coords, torch.zeros(R, 576 - 515, dtype=torch.float64)], -1)
    stacked = Lb @ U.T + torch.cat(c)
    for a in range(3):
        own = torch.cat([lat, coords[:, a:a + 1]], -1) @ u[a].T + c[a]
        assert torch.equal(stacked[:, 512 * a:512 * (a + 1)], own), a
        blk = U[512 * a:512 * (a + 1)]
        assert torch.equal(blk[:, :512], u[a][:, :512]) and torch.equal(blk[:, 512 + a], u[a][:, 512])
        others = [k for k in range(512, 576) if k != 512 + a]
        assert bool((blk[:, others] == 0).all())


def test_model_rounding_points():
    """With rounding on, every saved bf16 tensor of the model holds bf16 values, and the logits / planes are not rounded."""
    enc = small_encoder()
    nv, R = 1, G ** 3
    gen = torch.Generator().manual_seed(4)
    X = torch.randn(R, 518, generator=gen, dtype=torch.float64)
    planes, logits, S = tcm.forward(X, tcm.grid_coords(G, nv), tcm.params_of(enc), nv, G)
    for k in ("x", "h0", "h1", "lat", "Lb", "A"):
        assert torch.equal(S[k], tcm.bf(S[k])), k
    assert not torch.equal(logits, tcm.bf(logits))
    ups = [torch.randn(nv, 512, G, G, generator=gen, dtype=torch.float64) for _ in range(3)]
    mb = tcm.backward(*ups, S, tcm.params_of(enc), nv, G)
    assert not torch.equal(mb["g_X"], tcm.bf(mb["g_X"])) and not torch.equal(mb["d_logits"], tcm.bf(mb["d_logits"]))


@pytest.fixture(scope="module")
def lib():
    from neo360_b200 import build, _lib
    build.build()
    return _lib.load()


def test_tc_entry_points_reject_bad_arguments_without_gpu(lib):
    """The bf16 entry points of the encoder reject NULL buffers, nv < 1, strides and alignments their kernels cannot address -- all
    before any launch (the data pointers are never dereferenced)."""
    p = 1 << 20
    feat = lambda lat=p, nv=1, lh=4, lw=4, poses=p, X=p, ldx=576: lib.neo_grid_encoder_features_bf16(lat, nv, lh, lw, 8, 8, poses, 1.0, 0.0,
                                                                                                    0.0, X, ldx, None)
    for kw in (dict(lat=None), dict(poses=None), dict(X=None), dict(nv=0), dict(lh=1), dict(ldx=516), dict(ldx=520 + 4), dict(ldx=648),
               dict(lat=p + 4), dict(X=p + 8)):
        assert feat(**kw) == -1, kw
    assert b"neo_grid_encoder_features_bf16" in lib.neo_last_error()
    for args in ((None, 1, 576), (p, 0, 576), (p, 1, 512), (p, 1, 580), (p, 1, 648), (p + 8, 1, 576)):
        assert lib.neo_grid_encoder_coords_bf16(*args, None) == -1, args
    assert b"neo_grid_encoder_coords_bf16" in lib.neo_last_error()
    pool = lambda lat=p, ld=576, lg=p, nv=1, o=(p, p, p): lib.neo_grid_encoder_pool_bf16(lat, ld, lg, nv, *o, None)
    for kw in (dict(lat=None), dict(lg=None), dict(nv=0), dict(o=(p, None, p)), dict(ld=508), dict(ld=580), dict(lat=p + 8)):
        assert pool(**kw) == -1, kw
    assert b"neo_grid_encoder_pool_bf16" in lib.neo_last_error()
    pb = lambda lat=p, ld=576, lg=p, nv=1, dl=p, dg=p: lib.neo_grid_encoder_pool_bwd_bf16(lat, ld, lg, nv, None, None, None, dl, dg, None)
    for kw in (dict(lat=None), dict(lg=None), dict(nv=0), dict(dl=None), dict(dg=None), dict(ld=500)):
        assert pb(**kw) == -1, kw
    assert b"neo_grid_encoder_pool_bwd_bf16" in lib.neo_last_error()
    for args in ((None, p, 1, p), (p, None, 1, p), (p, p, 1, None), (p, p, 0, p), (p + 4, p, 1, p), (p, p + 8, 1, p), (p, p, 1, p + 4)):
        assert lib.neo_grid_encoder_lat_grad_bf16(*args, None) == -1, args
    assert b"neo_grid_encoder_lat_grad_bf16" in lib.neo_last_error()
