"""CPU: the float64 model of the tensor-core training form of the vanilla NeRF and Mip-NeRF 360 MLPs (oracle/dense_train_model.py).

* with its roundings off, the model equals vanilla._mlp_train and mip._mlp_train in float64 for all three MLP kinds;
* its hand-written adjoint equals autograd of the unrounded model to 1e-12;
* each bug of the mutation catalogue moves some output of the rounded model past twice the GPU bound, so the GPU tests would catch it.
"""
import pytest
import torch

from neo360_b200 import mip, vanilla
from oracle import dense_train_model as dtm

KINDS = ("vanilla", "prop", "mip")


def case(kind, n=6, N=5, seed=0):
    g = torch.Generator().manual_seed(seed)
    torch.manual_seed(seed)
    if kind == "vanilla":
        m, F = vanilla.NeRFMLP(), 63
    elif kind == "prop":
        m, F = mip.PropMLP(), 504
    else:
        m, F = mip.NeRFMLP(netwidth=128), 504
    m = m.double()
    with torch.no_grad():
        for p in m.parameters():
            p.add_(0.02 * torch.randn(p.shape, generator=g, dtype=torch.float64))
    feats = torch.randn(n * N, F, generator=g, dtype=torch.float64)
    denc = torch.randn(n, 27, generator=g, dtype=torch.float64)
    return m, feats, denc, n, N


@pytest.mark.parametrize("kind", KINDS)
def test_unrounded_model_is_mlp_train(kind):
    m, feats, denc, n, N = case(kind)
    P = dtm.params_of(m)
    sig, yb, _ = dtm.forward(feats, P, rnd=False)
    if kind == "vanilla":
        ref_rgb, ref_sig = vanilla._mlp_train(m, feats, denc, n, N)
        ref_sig = ref_sig.reshape(-1, 1)
    else:
        ref_sig, ref_rgb = mip._mlp_train(m, feats, denc, n, N)
        ref_sig = ref_sig.reshape(-1, 1)
    assert dtm.rel_err(sig, ref_sig) < 1e-12
    if kind == "prop":
        assert yb is None and ref_rgb is None
    else:
        assert dtm.rel_err(dtm.head(yb, denc, P, n, N), ref_rgb) < 1e-12


@pytest.mark.parametrize("kind", KINDS)
def test_adjoint_is_autograd(kind):
    m, feats, _, _, _ = case(kind, seed=1)
    P = dtm.params_of(m)
    leaves = {"w": [t.clone().requires_grad_(True) for t in P["w"]], "b": [t.clone().requires_grad_(True) for t in P["b"]]}
    Pg = dict(P, **leaves)
    for k in ("wsig", "bsig", "wb", "bb", "wvb"):
        if k in P:
            Pg[k] = P[k].clone().requires_grad_(True)
    sig, yb, S = dtm.forward(feats, Pg, rnd=False)
    gen = torch.Generator().manual_seed(5)
    gs = torch.randn(sig.shape, generator=gen, dtype=torch.float64)
    loss = (sig * gs).sum()
    gy = None
    if yb is not None:
        gy = torch.randn(yb.shape, generator=gen, dtype=torch.float64)
        loss = loss + (yb * gy).sum()
    loss.backward()
    det = lambda v: [t.detach() for t in v] if isinstance(v, list) else v.detach()
    G = dtm.backward(gs, gy, {k: det(v) for k, v in S.items()}, {k: det(v) for k, v in Pg.items()}, rnd=False)
    for i in range(len(P["w"])):
        assert dtm.rel_err(G[f"w{i}"], Pg["w"][i].grad) < 1e-12, i
        assert dtm.rel_err(G[f"b{i}"], Pg["b"][i].grad) < 1e-12, i
    for k in ("wsig", "bsig", "wb", "bb", "wvb"):
        if k in P:
            assert dtm.rel_err(G[k], Pg[k].grad) < 1e-12, k


@pytest.mark.parametrize("mut", dtm.MUTATIONS)
def test_mutations_exceed_bounds(mut):
    """Every planted bug moves an output past twice WIDE_FWD_BOUND or some gradient past twice WIDE_BWD_BOUND of the rounded model (the
    wide bounds are the looser ones)."""
    worst = 0.0
    for kind in KINDS:
        m, feats, _, _, _ = case(kind, n=20, N=8, seed=2)
        P = dtm.params_of(m)
        gen = torch.Generator().manual_seed(3)
        sig, yb, S = dtm.forward(feats, P)
        gs = 1e-2 * torch.randn(sig.shape, generator=gen, dtype=torch.float64)
        gy = None if yb is None else 1e-2 * torch.randn(yb.shape, generator=gen, dtype=torch.float64)
        G = dtm.backward(gs, gy, S, P)
        sig_m, yb_m, S_m = dtm.forward(feats, P, mut=mut)
        G_m = dtm.backward(gs, gy, S_m, P, mut=mut)
        worst = max(worst, dtm.rel_err(sig_m, sig) / dtm.WIDE_FWD_BOUND, *[dtm.rel_err(G_m[k], G[k]) / dtm.WIDE_BWD_BOUND for k in G])
        if yb is not None:
            worst = max(worst, dtm.rel_err(yb_m, yb) / dtm.WIDE_FWD_BOUND)
    assert worst > 2.0, (mut, worst)


def test_rounding_error_within_step_bound():
    """The bf16 roundings alone move the model by less than STEP_BOUND (the whole-step comparison against the fp32 path)."""
    for kind in KINDS:
        m, feats, _, _, _ = case(kind, n=40, N=10, seed=4)
        P = dtm.params_of(m)
        gen = torch.Generator().manual_seed(6)
        s_r, y_r, S_r = dtm.forward(feats, P)
        s_e, y_e, S_e = dtm.forward(feats, P, rnd=False)
        assert dtm.rel_err(s_r, s_e) < dtm.STEP_BOUND
        gs = torch.randn(s_r.shape, generator=gen, dtype=torch.float64)
        gy = None if y_r is None else torch.randn(y_r.shape, generator=gen, dtype=torch.float64)
        G_r, G_e = dtm.backward(gs, gy, S_r, P), dtm.backward(gs, gy, S_e, P, rnd=False)
        for k in G_r:
            assert dtm.rel_err(G_r[k], G_e[k]) < dtm.STEP_BOUND, (kind, k)
