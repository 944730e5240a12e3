"""CPU: the float64 restatement of the vanilla-NeRF compositing backward (oracle/vanilla_train_model.py, the arithmetic of
`neo_vanilla_composite_bwd`) against torch.autograd through `vanilla_oracle.composite` in float64, and the argument checks of the
vanilla training entry points (no GPU: the pointers are never dereferenced)."""
import pytest
import torch

from oracle import vanilla_oracle as vo
from oracle import vanilla_train_model as vtm

GRADS = ("g_comp", "g_acc", "g_w", "g_depth")


def composite_case(N, seed):
    """Ascending t in [2, 6] with non-unit |d| (0.3 .. 3): realistic sigma, a run of 6 opaque samples, an opaque first sample,
    all-zero sigma, duplicate t and a tiny sigma on the 1e10 interval."""
    g = torch.Generator().manual_seed(seed)
    n = 6
    t = 2.0 + 4.0 * torch.sort(torch.rand(n, N, generator=g, dtype=torch.float64), -1)[0]
    sig = torch.nn.functional.softplus(torch.randn(n, N, generator=g, dtype=torch.float64) * 2 - 1)
    if N >= 8:
        sig[1, 1:7] = 1e3
        t[4, 2:5] = t[4, 1]
    sig[2, 0] = 40.0 / max(float(t[2, 1] - t[2, 0]) if N > 1 else 1.0, 1e-3)
    sig[3] = 0.0
    sig[5, -1] = 1e-12
    rgb = torch.rand(n, N, 3, generator=g, dtype=torch.float64)
    d = torch.randn(n, 3, generator=g, dtype=torch.float64)
    d = d / d.norm(dim=-1, keepdim=True) * (0.3 + 2.7 * torch.rand(n, 1, generator=g, dtype=torch.float64))
    ups = {"g_comp": torch.randn(n, 3, generator=g, dtype=torch.float64), "g_acc": torch.randn(n, generator=g, dtype=torch.float64),
           "g_w": torch.randn(n, N, generator=g, dtype=torch.float64), "g_depth": torch.randn(n, generator=g, dtype=torch.float64)}
    return rgb, sig, t, d, ups


@pytest.mark.parametrize("N", [1, 2, 9, 40])
@pytest.mark.parametrize("white", [True, False], ids=["white", "black"])
def test_vanilla_composite_backward_equals_autograd(N, white):
    """Every upstream gradient alone and all together; N = 1 is the 1e10 interval alone."""
    rgb, sig, t, d, ups = composite_case(N, 11 * N + white)
    for use in [[k] for k in GRADS] + [list(GRADS)]:
        r, s = rgb.clone().requires_grad_(True), sig.clone().requires_grad_(True)
        comp, acc, w, depth = vo.composite(r, s[..., None], t, d, white)
        outs = {"g_comp": comp, "g_acc": acc, "g_w": w, "g_depth": depth}
        loss = sum((outs[k] * ups[k]).sum() for k in use)
        gr, gs = torch.autograd.grad(loss, [r, s], allow_unused=True, materialize_grads=True)
        m = vtm.composite_bwd(rgb, sig, t, d, white, fp32=False, **{k: ups[k] for k in use})
        for got, ref, mag in ((m["d_sigma"], gs, m["d_sigma_mag"]), (m["d_rgb"], gr, m["d_rgb_mag"])):
            err = (got - ref).abs()
            assert bool((err <= 1e-12 * mag + 1e-300).all()), (use, float((err / mag.clamp_min(1e-300)).max()))
    f = vtm.composite_fwd(rgb, sig, t, d, white, fp32=False)
    comp, acc, w, depth = vo.composite(rgb, sig[..., None], t, d, white)
    for a, b in ((f["comp"], comp), (f["acc"], acc), (f["w"], w), (f["depth"], depth)):
        assert float((a - b).abs().max()) <= 1e-13 * max(1.0, float(t.abs().max()))


def test_vanilla_composite_fp32_model_rounds_like_the_kernel():
    """fp32 on: the interval is the fp32 product fp32(t_{k+1} - t_k) * fp32 |d|, the last one fp32(1e10 |d|); off: float64."""
    t = torch.tensor([[2.0, 2.1, 2.3]], dtype=torch.float64)
    d = torch.tensor([[0.6, 0.0, 0.8]], dtype=torch.float64) * 1.7
    sig = torch.tensor([[0.5, 0.5, 0.5]], dtype=torch.float64)
    k32, k64 = vtm.composite_terms(sig, t, d, fp32=True), vtm.composite_terms(sig, t, d, fp32=False)
    dn32 = torch.linalg.norm(d.float(), dim=-1)
    want = torch.stack([(t.float()[0, 1] - t.float()[0, 0]) * dn32[0], (t.float()[0, 2] - t.float()[0, 1]) * dn32[0], 1e10 * dn32[0]])
    assert torch.equal(k32["dist"][0], want.double())
    assert float((k64["dist"][0] - torch.tensor([0.1, 0.2, 1e10], dtype=torch.float64) * 1.7).abs().max()) < 1e-6


@pytest.fixture(scope="module")
def lib():
    from neo360_b200 import build, _lib
    build.build()
    return _lib.load()


def test_vanilla_training_entry_points_validate_arguments_without_gpu(lib):
    """The three new entry points are exported and reject NULL inputs / outputs, n <= 0 and N < 1 (n_coarse < 1) before any launch."""
    from neo360_b200 import _lib as L
    for name in ("neo_vanilla_sample_along_rays", "neo_vanilla_encode", "neo_vanilla_composite_bwd"):
        assert name in L.SYMBOLS and hasattr(lib, name)
    p = 1 << 20
    smp = lambda o, vd, n, nc, t: lib.neo_vanilla_sample_along_rays(o, vd, n, nc, 2.0, 6.0, None, t, None)
    for args in ((None, p, 4, 8, p), (p, None, 4, 8, p), (p, p, 4, 8, None), (p, p, 0, 8, p), (p, p, -3, 8, p), (p, p, 4, 0, p)):
        assert smp(*args) == -1, args
    assert b"neo_vanilla_sample_along_rays" in lib.neo_last_error()
    enc = lambda o, vd, t, n, N, e, de: lib.neo_vanilla_encode(o, vd, t, n, N, e, de, None)
    for args in ((None, p, p, 4, 8, p, p), (p, None, p, 4, 8, p, p), (p, p, None, 4, 8, p, p), (p, p, p, 4, 8, None, p),
                 (p, p, p, 4, 8, p, None), (p, p, p, 0, 8, p, p), (p, p, p, 4, 0, p, p)):
        assert enc(*args) == -1, args
    assert b"neo_vanilla_encode" in lib.neo_last_error()
    bwd = lambda rgb, sig, t, d, n, N, dr, ds: lib.neo_vanilla_composite_bwd(rgb, sig, t, d, n, N, 1, p, None, None, None, dr, ds, None)
    for args in ((None, p, p, p, 4, 8, p, p), (p, None, p, p, 4, 8, p, p), (p, p, None, p, 4, 8, p, p), (p, p, p, None, 4, 8, p, p),
                 (p, p, p, p, 4, 8, None, p), (p, p, p, p, 4, 8, p, None), (p, p, p, p, 0, 8, p, p), (p, p, p, p, -1, 8, p, p),
                 (p, p, p, p, 4, 0, p, p)):
        assert bwd(*args) == -1, args
    assert b"neo_vanilla_composite_bwd" in lib.neo_last_error()


def test_training_mlp_equals_the_oracle_mlp_in_float64():
    """vanilla._mlp_train (the framework layers of the training path, dir_enc columns of views_linear.0 applied once per ray) equals
    `vanilla_oracle.mlp_forward` in float64, values and parameter gradients."""
    from neo360_b200 import synth
    from neo360_b200.vanilla import NeRF, _mlp_train
    Pm = {k: v.double() for k, v in synth.make_vanilla_params(4).items()}
    net = NeRF(num_coarse_samples=8, num_fine_samples=4).double()
    net.load_state_dict(Pm)
    g = torch.Generator().manual_seed(0)
    n, N = 5, 7
    enc, denc = torch.randn(n * N, 63, generator=g, dtype=torch.float64), torch.randn(n, 27, generator=g, dtype=torch.float64)
    Pg = {k: v.clone().requires_grad_(True) for k, v in Pm.items()}
    rgb_r, sig_r = vo.mlp_forward(Pg, "fine_mlp.", enc.reshape(n, N, 63), denc)
    rgb, sig = _mlp_train(net.fine_mlp, enc, denc, n, N)
    assert float((rgb - rgb_r).detach().abs().max()) < 1e-12 and float((sig - sig_r).detach().abs().max()) < 1e-12
    (rgb_r.sin().sum() + sig_r.cos().sum()).backward()
    (rgb.sin().sum() + sig.cos().sum()).backward()
    for name, p in net.fine_mlp.named_parameters():
        ref = Pg["fine_mlp." + name].grad
        assert float((p.grad - ref).abs().max()) <= 1e-12 * max(1.0, float(ref.abs().max())), name
