"""CPU: the models of the deterministic training kernels (oracle/det_model.py) against autograd through the library's own framework
forms, their mutation catalogue, and the new entry points' argument checks (no GPU needed)."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from neo360_b200 import mip, training
from oracle import det_model as dm

torch.set_default_dtype(torch.float32)


def ray_batch(n, N, seed, descending=False, zero_rows=0):
    g = torch.Generator().manual_seed(seed)
    w = torch.rand(n, N, generator=g, dtype=torch.float64) ** 3
    w[:zero_rows] = 0
    m = torch.sort(torch.rand(n, N, generator=g, dtype=torch.float64), -1, descending=descending).values
    I = torch.rand(n, N, generator=g, dtype=torch.float64) / N
    return w, m, I


@pytest.mark.parametrize("descending", [False, True], ids=["fg ascending m", "bg descending m"])
@pytest.mark.parametrize("N", [1, 2, 33, 129])
def test_distortion_float64_equals_autograd(N, descending):
    w, m, I = ray_batch(7, N, N, descending, zero_rows=1)
    wl = w.clone().requires_grad_(True)
    g = torch.rand(7, dtype=torch.float64)
    per_ray = dm.distortion64(wl, m, I)
    # training.distortion_loss is the mean over rays of the same functional
    assert abs(float(per_ray.detach().mean() - training.distortion_loss(w, m, I))) < 1e-12
    (per_ray * g).sum().backward()
    assert float((wl.grad - dm.distortion_grad64(w, m, I, g)).abs().max()) < 1e-12


def test_distortion_descending_m_is_minus_the_pair_form():
    """The formula as written, with bg's descending m, gives minus sum w_i w_j |m_i - m_j| for the pair term (as the reference does)."""
    w, m, I = ray_batch(3, 17, 5, descending=True)
    pair = (w[:, :, None] * w[:, None, :] * (m[:, :, None] - m[:, None, :]).abs()).sum((-1, -2))
    got = dm.distortion64(w, m, torch.zeros_like(I))
    assert float((got + pair).abs().max()) < 1e-12


def mip_levels(n, Nc, Np, seed, ties=False):
    g = torch.Generator().manual_seed(seed)
    c = torch.sort(torch.rand(n, Nc + 1, generator=g), -1).values
    te = torch.sort(torch.rand(n, Np + 1, generator=g), -1).values
    if ties and Np >= 6:
        te[:, 3:6] = te[:, 3:4]                         # tied knots: empty envelope intervals
        c[:, 2] = te[:, 3]                               # an sdist on a knot
        c[:, 0], c[:, -1] = -0.1, 1.1                     # outside the envelope
        c = torch.sort(c, -1).values                      # the NeRF level's sdist ascends
    w = torch.rand(n, Nc, generator=g) ** 2
    we = torch.rand(n, Np, generator=g) ** 2
    we[:, Np // 2] = 0
    return c.double(), w.double(), te.double(), we.double()


@pytest.mark.parametrize("ties", [False, True])
@pytest.mark.parametrize("Nc,Np", [(1, 1), (8, 16), (32, 64)])
def test_interlevel_float64_equals_autograd(Nc, Np, ties):
    c, w, te, we = mip_levels(5, Nc, Np, Nc + Np, ties)
    wl = we.clone().requires_grad_(True)
    ref = (torch.clip(w - mip._outer_weights(c, te, wl), min=0) ** 2 / (w + dm.EPS))
    assert float((ref.mean(-1) - dm.interlevel64(c, w, te, we)).abs().max()) < 1e-12
    g = torch.rand(5, dtype=torch.float64)
    (ref.mean(-1) * g).sum().backward()
    assert float((wl.grad - dm.interlevel_grad64(c, w, te, we, g)).abs().max()) < 1e-12


SHAPES = [((16, 16), (32, 32)), ((32, 32), (120, 160)), ((240, 320), (240, 320)), ((15, 20), (240, 320)), ((1, 5), (3, 7)), ((4, 4), (1, 1))]


@pytest.mark.parametrize("hw_in,hw_out", SHAPES)
def test_upsample_adjoint(hw_in, hw_out):
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 3, *hw_in, generator=g, dtype=torch.float64)
    y = torch.randn(2, 3, *hw_out, generator=g, dtype=torch.float64)
    up = F.interpolate(x, hw_out, mode="bilinear", align_corners=True)
    assert float((up - dm.upsample64(x, hw_out, fp32=False)).abs().max()) < 1e-12
    assert abs(float((dm.upsample64(x, hw_out) * y).sum() - (x * dm.upsample_adjoint64(y, hw_in)).sum())) < 1e-9
    xl = x.clone().requires_grad_(True)
    (F.interpolate(xl, hw_out, mode="bilinear", align_corners=True) * y).sum().backward()
    assert float((xl.grad - dm.upsample_adjoint64(y, hw_in, fp32=False)).abs().max()) < 1e-12
    # the fp32 weights are ATen's fp32 forward's: the float32 framework forward agrees with the fp32-weight model to fp32 rounding
    up32 = F.interpolate(x.float(), hw_out, mode="bilinear", align_corners=True)
    assert float((up32.double() - dm.upsample64(x.float(), hw_out)).abs().max()) < 1e-5


def test_segment_emulation_within_bound_and_order_matters():
    g = torch.Generator().manual_seed(3)
    E, T, C = 5000, 40, 8
    keys = torch.randint(0, T + 1, (E,), generator=g)
    wts = torch.rand(E, generator=g)
    rows = torch.randn(E, C, generator=g) * torch.exp(torch.randn(E, 1, generator=g) * 4)
    order = torch.argsort(keys, stable=True)
    ks, ids = keys[order], order
    g_of = lambda e: rows[e]
    init = torch.randn(T, C, generator=g)
    got = dm.segment_emulate(ks, ids, wts, g_of, init)
    val, mag, n = dm.scatter_exact(ks, ids, wts, g_of, init)
    assert bool(((got.double() - val).abs() <= dm.scatter_bound(mag, n)).all())
    rev = dm.segment_emulate(ks, ids, wts, g_of, init, reverse=True)
    assert not torch.equal(rev, got)
    assert torch.equal(dm.segment_emulate(ks, ids, wts, g_of, init), got)


def test_mutation_catalogue():
    """Each planted defect of a model moves its result far outside the bound the kernels are held to (printed as a multiple of it)."""
    w, m, I = ray_batch(16, 65, 11, descending=True)
    abs_pair = lambda w, m, I: (I * w * w).sum(-1) / 3 + (w[:, :, None] * w[:, None, :] * (m[:, :, None] - m[:, None, :]).abs()).sum((-1, -2))
    lb, _ = dm.distortion_bounds(w, m, I, torch.ones(16))
    d1 = float(((abs_pair(w, m, I) - dm.distortion64(w, m, I)).abs() / lb).max())
    c, wn, te, we = mip_levels(16, 32, 64, 2)
    il, _ = dm.interlevel_bounds(c, wn, te, we, torch.ones(16))
    d2 = float(((dm.interlevel64(c, wn, te, we, short=True) - dm.interlevel64(c, wn, te, we)).abs() / il).max())
    gy = torch.randn(1, 1, 32, 32, dtype=torch.float64)
    ub = dm.upsample_bound(gy, (16, 16))
    d3 = float(((dm.upsample_adjoint64(gy, (16, 16), short=True) - dm.upsample_adjoint64(gy, (16, 16))).abs() / ub).max())
    print(f"distortion with |m_i - m_j|: {d1:.3g} x bound; interlevel over [lo_j, hi_j): {d2:.3g} x bound; "
          f"upsample gather one row short: {d3:.3g} x bound")
    assert min(d1, d2, d3) > 100


@pytest.fixture(scope="module")
def lib():
    from neo360_b200 import build, _lib
    build.build()
    return _lib.load()


def test_argument_checks_without_gpu(lib):
    p = 1 << 20
    sc = p                                              # never dereferenced: every call below fails its checks first
    assert lib.neo_index_maps_bwd_det(sc, p, 8, 6, p, None, p, None, None, None, p, 1 << 30, None) == -1     # C % 4
    assert lib.neo_index_maps_bwd_det(sc, p, 8, 256, p + 4, None, p, None, None, None, p, 1 << 30, None) == -1  # g_local alignment
    assert lib.neo_index_maps_bwd_det(sc, p, 8, 256, p, None, p, None, None, None, None, 1 << 30, None) == -1  # no workspace
    assert lib.neo_index_maps_bwd_det(sc, p, 8, 256, p, None, p, None, None, None, p + 8, 1 << 30, None) == -1  # workspace alignment
    assert lib.neo_index_maps_bwd_det(sc, p, 8, 256, None, p, None, p, None, p, p, 1 << 30, None) == -1      # a NULL plane
    assert lib.neo_index_maps_bwd_det_workspace_bytes(None, 8, 256) == 0
    assert lib.neo_index_maps_bwd_det_workspace_bytes(sc, 8, 6) == 0
    f = lambda **k: lib.neo_grid_encoder_features_bwd_det(k.get("nv", 1), 4, 4, 8, 8, p, 1.0, 0.0, 0.0, k.get("g", p), k.get("ldg", 518),
                                                          k.get("gl", p), k.get("ws", p), 1 << 30, None)
    assert f(nv=0) == -1 and f(g=None) == -1 and f(ldg=511) == -1 and f(ldg=519) == -1 and f(gl=p + 4) == -1 and f(ws=None) == -1
    assert f(ws=p + 4) == -1
    assert b"neo_grid_encoder_features_bwd_det" in lib.neo_last_error()
    assert lib.neo_grid_encoder_features_bwd_det_workspace_bytes(0, 4, 4) == 0
    assert lib.neo_distortion_loss(None, p, None, 0.0, 4, 4, p, None) == -1
    assert lib.neo_distortion_loss(p, p, None, 0.0, 0, 4, p, None) == -1
    assert lib.neo_distortion_loss_bwd(p, p, None, 0.0, 4, 4, p, None, None) == -1
    assert lib.neo_interlevel_loss(p, p, p, p, 4, 0, 8, p, None) == -1
    assert lib.neo_interlevel_loss(p, p, p, p, 4, 1025, 8, p, None) == -1
    assert lib.neo_interlevel_loss_bwd(p, p, p, None, 4, 4, 8, p, p, None) == -1
    assert lib.neo_upsample_bilinear_bwd(p, 1, 0, 4, 8, 8, p, None) == -1
    assert lib.neo_upsample_bilinear_bwd(None, 1, 4, 4, 8, 8, p, None) == -1
    assert b"neo_upsample_bilinear_bwd" in lib.neo_last_error()
