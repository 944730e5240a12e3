"""CPU: the float64 model of the PixelNeRF form of the tensor-core training trunk (oracle/pixelnerf_train_tc_model.py), which the GPU
tests of `PixelNeRF(train_precision="tc")` hold the kernels to.

* with its roundings off, the projection (p0 = latent rows . W0[:, 63:575]^T), the trunk and the per-point head equal
  pixelnerf._mlp_train (the reference formulation, per-view head) in float64;
* its hand-written adjoint equals autograd of the unrounded model to 1e-12;
* each bug only this form can have moves some output of the rounded model past twice its GPU bound;
* the bf16 roundings alone stay within STEP_BOUND, the bound of the whole-step comparison against the "fp32" path.
"""
import pytest
import torch

from neo360_b200 import pixelnerf
from oracle import pixelnerf_train_tc_model as ptm


def case(nv=3, M=40, seed=0):
    g = torch.Generator().manual_seed(seed)
    torch.manual_seed(seed)
    mlp = pixelnerf.NeRFMLP().double()
    with torch.no_grad():
        for p in mlp.parameters():
            p.add_(0.05 * torch.randn(p.shape, generator=g, dtype=torch.float64))
    cam = torch.randn(nv, M, 3, generator=g, dtype=torch.float64)
    local = 0.3 * torch.randn(nv * M, 512, generator=g, dtype=torch.float64)      # looked-up latent rows
    dir_tile = torch.randn(nv * M, 27, generator=g, dtype=torch.float64)
    return mlp, cam, local, dir_tile


def run(mlp, cam, local, dir_tile, g, rnd=True, mut=None):
    """Projection, trunk, head and the trunk's adjoint of the model -> dict of every tensor the GPU tests compare."""
    nv = cam.shape[0]
    W = ptm.weights_of(mlp)
    p0 = ptm.project(local, mlp.pts_linears[0].weight.detach(), mut=mut)
    hbar, S = ptm.forward(cam, p0, W, rnd=rnd, mut=mut)
    rgb, sigma = ptm.head(mlp, hbar, dir_tile, nv, mut=mut)
    d_p0, G = ptm.backward(g, S, W, rnd=rnd, mut=mut)
    return dict(hbar=hbar, rgb=rgb.detach(), sigma=sigma.detach(), d_p0=d_p0, **G)


def test_weights_are_the_pixel_form():
    W = ptm.weights_of(pixelnerf.NeRFMLP())
    assert "w3e" not in W and W["w3"].shape == (128, 128) and W["w0e"].shape == (128, 63)


@pytest.mark.parametrize("nv", [1, 3])
def test_unrounded_model_is_mlp_train(nv):
    mlp, cam, local, dir_tile = case(nv)
    enc = ptm.pos_enc(cam).reshape(-1, 63)
    ref_rgb, ref_sigma = pixelnerf._mlp_train(mlp, enc, dir_tile, local, nv)
    p0 = ptm.project(local, mlp.pts_linears[0].weight.detach())
    hbar, _ = ptm.forward(cam, p0, ptm.weights_of(mlp), rnd=False)
    rgb, sigma = ptm.head(mlp, hbar, dir_tile, nv)
    assert ptm.rel_err(rgb, ref_rgb) < 1e-12
    assert ptm.rel_err(sigma, ref_sigma) < 1e-12


def test_adjoint_is_autograd():
    nv = 2
    mlp, cam, local, _ = case(nv, seed=1)
    W = {k: v.clone().requires_grad_(True) for k, v in ptm.weights_of(mlp).items()}
    p0 = ptm.project(local, mlp.pts_linears[0].weight.detach()).requires_grad_(True)
    hbar, S = ptm.forward(cam, p0, W, rnd=False)
    g = torch.randn(hbar.shape, generator=torch.Generator().manual_seed(5), dtype=torch.float64)
    (hbar * g).sum().backward()
    d_p0, G = ptm.backward(g, {k: (v.detach() if torch.is_tensor(v) else v) for k, v in S.items()},
                           {k: v.detach() for k, v in W.items()}, rnd=False)
    assert ptm.rel_err(d_p0, p0.grad) < 1e-12
    assert set(G) == set(W)
    for k in W:
        assert ptm.rel_err(G[k], W[k].grad) < 1e-12, k


@pytest.mark.parametrize("mut", ptm.MUTATIONS)
def test_mutations_exceed_bounds(mut):
    """Every planted bug moves hbar, rgb or sigma past FWD_BOUND or some gradient past BWD_BOUND of the rounded model, by 2x."""
    mlp, cam, local, dir_tile = case(3, seed=2)
    g = torch.randn(cam.shape[1], 128, generator=torch.Generator().manual_seed(3), dtype=torch.float64)
    ok, bad = run(mlp, cam, local, dir_tile, g), run(mlp, cam, local, dir_tile, g, mut=mut)
    fwd = ("hbar", "rgb", "sigma")
    worst = max(ptm.rel_err(bad[k], ok[k]) / (ptm.FWD_BOUND if k in fwd else ptm.BWD_BOUND) for k in ok)
    assert worst > 2.0, (mut, worst)


def test_rounding_error_within_step_bound():
    """The bf16 roundings alone move every output of the model by less than STEP_BOUND."""
    mlp, cam, local, dir_tile = case(3, M=400, seed=4)
    g = torch.randn(400, 128, generator=torch.Generator().manual_seed(6), dtype=torch.float64)
    rounded, exact = run(mlp, cam, local, dir_tile, g), run(mlp, cam, local, dir_tile, g, rnd=False)
    for k in exact:
        assert ptm.rel_err(rounded[k], exact[k]) < ptm.STEP_BOUND, k
