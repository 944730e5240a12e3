"""CPU: the float64 model of the tensor-core training trunk (oracle/field_train_model.py).

* with its roundings off, the model's trunk and head equal training._mlp_projected in float64, for the foreground (in_ch 3) and the
  background (in_ch 4) MLP;
* its hand-written adjoint equals autograd of the unrounded model to 1e-12;
* each value-level bug of the mutation catalogue moves some output of the rounded model by more than the GPU bound, so the GPU tests
  would catch it.
"""
import pytest
import torch

from neo360_b200 import training
from neo360_b200.renderer import NeRFPPMLP
from oracle import field_train_model as ftm


def case(ich, nv=3, M=40, seed=0):
    g = torch.Generator().manual_seed(seed)
    torch.manual_seed(seed)
    mlp = NeRFPPMLP(0, 10, 4, num_src_views=nv, input_ch=ich).double()
    with torch.no_grad():
        for p in mlp.parameters():
            p.add_(0.05 * torch.randn(p.shape, generator=g, dtype=torch.float64))
    cam = torch.randn(nv, M, ich, generator=g, dtype=torch.float64)
    lp = 0.3 * torch.randn(nv * M, 256, generator=g, dtype=torch.float64)
    wp = 0.3 * torch.randn(nv * M, 256, generator=g, dtype=torch.float64)
    dir_tile = torch.randn(nv * M, 27, generator=g, dtype=torch.float64)
    return mlp, cam, lp, wp, dir_tile


@pytest.mark.parametrize("ich", [3, 4])
def test_unrounded_model_is_mlp_projected(ich):
    nv = 3
    mlp, cam, lp, wp, dir_tile = case(ich, nv)
    ref_rgb, ref_sigma = training._mlp_projected(mlp, training._pos_enc(cam, 0, 10), dir_tile, lp, wp, nv)
    hbar, _ = ftm.forward(cam, lp, wp, ftm.weights_of(mlp, ich), rnd=False)
    rgb, sigma = ftm.head(mlp, hbar, dir_tile, nv)
    assert ftm.rel_err(rgb, ref_rgb) < 1e-12
    assert ftm.rel_err(sigma, ref_sigma) < 1e-12


@pytest.mark.parametrize("ich", [3, 4])
def test_adjoint_is_autograd(ich):
    nv = 2
    mlp, cam, lp, wp, _ = case(ich, nv, seed=1)
    W = {k: v.clone().requires_grad_(True) for k, v in ftm.weights_of(mlp, ich).items()}
    lp, wp = lp.clone().requires_grad_(True), wp.clone().requires_grad_(True)
    hbar, S = ftm.forward(cam, lp, wp, W, rnd=False)
    g = torch.randn(hbar.shape, generator=torch.Generator().manual_seed(5), dtype=torch.float64)
    (hbar * g).sum().backward()
    d_pm, G = ftm.backward(g, {k: (v.detach() if torch.is_tensor(v) else v) for k, v in S.items()},
                           {k: v.detach() for k, v in W.items()}, rnd=False)
    assert ftm.rel_err(d_pm, lp.grad) < 1e-12 and ftm.rel_err(d_pm, wp.grad) < 1e-12
    for k in W:
        assert ftm.rel_err(G[k], W[k].grad) < 1e-12, k


@pytest.mark.parametrize("mut", ftm.MUTATIONS)
def test_mutations_exceed_bounds(mut):
    """Every planted bug moves hbar past FWD_BOUND or some gradient past BWD_BOUND of the rounded model."""
    worst = 0.0
    for ich in (3, 4):
        mlp, cam, lp, wp, _ = case(ich, 3, seed=2)
        W = ftm.weights_of(mlp, ich)
        g = torch.randn(cam.shape[1], 128, generator=torch.Generator().manual_seed(3), dtype=torch.float64)
        hbar, S = ftm.forward(cam, lp, wp, W)
        d_pm, G = ftm.backward(g, S, W)
        hbar_m, S_m = ftm.forward(cam, lp, wp, W, mut=mut)
        d_pm_m, G_m = ftm.backward(g, S_m, W, mut=mut)
        worst = max(worst, ftm.rel_err(hbar_m, hbar) / ftm.FWD_BOUND, ftm.rel_err(d_pm_m, d_pm) / ftm.BWD_BOUND,
                    *[ftm.rel_err(G_m[k], G[k]) / ftm.BWD_BOUND for k in G])
    assert worst > 2.0, (mut, worst)


def test_rounding_error_within_step_bound():
    """The bf16 roundings alone move the model by less than STEP_BOUND (the whole-step comparison against the fp32 path)."""
    for ich in (3, 4):
        mlp, cam, lp, wp, _ = case(ich, 3, M=400, seed=4)
        W = ftm.weights_of(mlp, ich)
        g = torch.randn(cam.shape[1], 128, generator=torch.Generator().manual_seed(6), dtype=torch.float64)
        h_r, S_r = ftm.forward(cam, lp, wp, W)
        h_e, S_e = ftm.forward(cam, lp, wp, W, rnd=False)
        assert ftm.rel_err(h_r, h_e) < ftm.STEP_BOUND
        d_r, G_r = ftm.backward(g, S_r, W)
        d_e, G_e = ftm.backward(g, S_e, W, rnd=False)
        assert ftm.rel_err(d_r, d_e) < ftm.STEP_BOUND
        for k in G_r:
            assert ftm.rel_err(G_r[k], G_e[k]) < ftm.STEP_BOUND, k
