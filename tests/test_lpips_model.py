"""CPU: the float64 LPIPS models of oracle/lpips_model.py, their bounds, weight loading and the patch order of the fine-tuning batch.

* piqa's and lpips' definitions agree to 1e-12 in float64; LPIPS(x, x) = 0 and LPIPS is symmetric.
* the head's adjoint equals autograd through the float64 model behind a ReLU, zero-norm pixels included.
* `LPIPS.from_files` reads torchvision's vgg16 layout and both lin layouts, and names a missing, unknown or mis-shaped key.
* `batches.patch_pix_inds` lists the 30x30 patch as `view(H, W)[x:x+30, y:y+30].reshape(-1)` does, at the four corners.
* a catalogue of model mutants each lands far outside the bounds the GPU tests hold the kernels to.
"""
import numpy as np
import pytest
import torch

from oracle import lpips_model as lm


def frames(n, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return 1.2 * torch.rand(n, H, W, 3, generator=g, dtype=torch.float64) - 0.1, torch.rand(n, H, W, 3, generator=g, dtype=torch.float64)


@pytest.fixture(scope="module")
def vgg():
    return lm.vgg16_state(0)


@pytest.fixture(scope="module")
def feats(vgg):
    """Float64 trunk features of two frame pairs at 37x53 with planted zero-norm and tiny-norm pixels."""
    x, y = frames(2, 37, 53, 1)
    fx = lm.plant(lm.trunk_f64(vgg, lm.scale_f64(x, 0)), seed=1, zero_frac=0.1)
    fy = lm.plant(lm.trunk_f64(vgg, lm.scale_f64(y, 0)), seed=2, zero_frac=0.1)
    return fx, fy, lm.lin_weights(0)


@pytest.mark.parametrize("H,W", [(32, 32), (37, 53)])
def test_piqa_and_lpips_definitions_agree(vgg, H, W):
    x, y = frames(2, H, W, H + W)
    ws = lm.lin_weights(1)
    a, b = lm.lpips_piqa_f64(x, y, vgg, ws), lm.lpips_lpips_f64(x, y, vgg, ws)
    assert (a > 0).all()
    assert float((a - b).abs().max()) <= 1e-12 * float(a.abs().max())


def test_identical_is_zero_and_symmetric(vgg):
    x, y = frames(2, 32, 40, 5)
    ws = lm.lin_weights(2)
    assert (lm.lpips_piqa_f64(x, x, vgg, ws) == 0).all()
    assert torch.allclose(lm.lpips_lpips_f64(x, y, vgg, ws), lm.lpips_lpips_f64(y, x, vgg, ws), rtol=1e-14, atol=0)


def test_adjoint_matches_autograd_behind_relu(feats):
    fx, fy, ws = feats
    g = torch.tensor([0.7, -1.3], dtype=torch.float64)
    # pre-activations whose ReLU gives the planted features: zero-norm pixels have every channel <= 0
    zx = [torch.where(f > 0, f, -torch.rand_like(f)).requires_grad_(True) for f in fx]
    zy = [torch.where(f > 0, f, -torch.rand_like(f)).requires_grad_(True) for f in fy]
    val = lm.head_f64([torch.relu(z) for z in zx], [torch.relu(z) for z in zy], ws)[0]
    (val * g).sum().backward()
    gx, gy = lm.adjoint_f64(fx, fy, ws, g)
    for k in range(5):
        zero = (fx[k] * fx[k]).sum(1) == 0
        assert zero.any(), k
        for z, a in ((zx[k], gx[k]), (zy[k], gy[k])):
            ref = z.grad
            assert torch.isfinite(ref).all()
            got = a * (z > 0)
            assert float((got - ref).abs().max()) <= 1e-12 * float(ref.abs().max()), k
        assert (gx[k].permute(0, 2, 3, 1)[zero] == 0).all()


def test_bounds_cover_the_framework_form_in_fp32(feats):
    """head_torch in fp32 (another summation order) stays inside the head bound: the bound is not tighter than fp32 arithmetic allows."""
    from neo360_b200.lpips import head_torch
    fx, fy, ws = feats
    ref, _ = lm.head_f64(fx, fy, ws)
    bound, _ = lm.head_bound(fx, fy, ws)
    got = head_torch([f.float() for f in fx], [f.float() for f in fy], ws).double()
    r = float(((got - ref).abs() / bound).max())
    print(f"framework fp32 form: {r:.3g} of the bound")
    assert r <= 1


def test_mutants_leave_the_bounds(feats):
    fx, fy, ws = feats
    ref, per = lm.head_f64(fx, fy, ws)
    bound, per_bound = lm.head_bound(fx, fy, ws)

    def far(v, b):
        r = ((v - ref).abs() / b)
        return bool(torch.isnan(v).any()) or float(r.max()) > 100

    # eps dropped: zero-norm pixels become NaN, and the tiny-norm ones move
    assert far(lm.head_f64(fx, fy, ws, eps=0.0)[0], bound)
    no_zero_x = [torch.where((f * f).sum(1, keepdim=True) == 0, torch.full_like(f, 1e-12), f) for f in fx]
    no_zero_y = [torch.where((f * f).sum(1, keepdim=True) == 0, torch.full_like(f, 1e-12), f) for f in fy]
    r0 = lm.head_f64(no_zero_x, no_zero_y, ws)[0]
    assert far(lm.head_f64(no_zero_x, no_zero_y, ws, eps=0.0)[0] - r0 + ref, lm.head_bound(no_zero_x, no_zero_y, ws)[0])
    # layer weights: rolled by one channel, and the two 512-channel layers exchanged
    assert far(lm.head_f64(fx, fy, [torch.roll(w, 1) for w in ws])[0], bound)
    swapped = lm.head_f64(fx, fy, ws[:3] + [ws[4], ws[3]])[1]
    assert float(((swapped - per).abs() / per_bound).max()) > 100
    # mean over the frame's H W instead of the layer's
    P0 = fx[0].shape[2] * fx[0].shape[3]
    wrong = sum(per[:, k] * fx[k].shape[2] * fx[k].shape[3] / P0 for k in range(5))
    assert far(wrong, bound)
    # the norm short one group of 4 channels
    short = 0
    for a, b, w in zip(fx, fy, ws):
        u = a / (torch.sqrt((a[:, :-4] ** 2).sum(1, keepdim=True)) + lm.EPS)
        v = b / (torch.sqrt((b[:, :-4] ** 2).sum(1, keepdim=True)) + lm.EPS)
        short = short + (w.double().reshape(1, -1, 1, 1) * (u - v) ** 2).sum(1).mean((1, 2))
    assert far(short, bound)
    # backward without the projection term
    g = torch.tensor([1.0, 0.5], dtype=torch.float64)
    gx, _ = lm.adjoint_f64(fx, fy, ws, g)
    mx, _ = lm.adjoint_f64(fx, fy, ws, g, projection=False)
    bx, _ = lm.bwd_bound(fx, fy, ws, g)
    assert max(float(((m - a).abs() / b.clamp_min(1e-300)).max()) for m, a, b in zip(mx, gx, bx)) > 100


def test_prepare_emulation_against_float64():
    g = torch.Generator().manual_seed(3)
    x = (1.4 * torch.rand(2, 5, 7, 3, generator=g) - 0.2).numpy()
    for form in (0, 1):
        got = lm.prepare_f32(x, form).astype(np.float64)
        ref = lm.scale_f64(torch.from_numpy(x), form).numpy()
        assert np.abs(got - ref).max() <= 4 * 2.0 ** -24 * np.abs(ref).max()
        gout = np.random.default_rng(form).standard_normal((2, 3, 5, 7)).astype(np.float32)
        gi = lm.prepare_bwd_f32(x, gout, form)
        inside = (x >= 0) & (x <= 1)
        assert (gi[~inside] == 0).all()
        scale = np.asarray(lm.STD if form == 0 else [s / 2 for s in lm.SCALE])
        assert np.allclose(gi[inside], (gout.transpose(0, 2, 3, 1) / scale)[inside], rtol=1e-6)


@pytest.mark.parametrize("layout", ["lpips", "piqa"])
def test_from_files_layouts(tmp_path, vgg, layout):
    from neo360_b200.lpips import LPIPS
    ws = lm.lin_weights(4)
    torch.save(vgg, tmp_path / "vgg16.pth")
    torch.save(lm.lin_state(ws, layout), tmp_path / "vgg.pth")
    m = LPIPS.from_files(str(tmp_path / "vgg16.pth"), str(tmp_path / "vgg.pth"))
    for k in range(5):
        assert torch.equal(m.lin[k], ws[k])
    for i in lm.CONVS:
        assert torch.equal(m.features[i].weight, vgg[f"features.{i}.weight"]) and torch.equal(m.features[i].bias, vgg[f"features.{i}.bias"])
    assert not any(p.requires_grad for p in m.parameters())
    x = lm.scale_f64(frames(1, 32, 32, 9)[0], 0)
    for a, b in zip(m.trunk(x.float()), lm.trunk_f64(vgg, x)):
        assert a.shape == b.shape and float((a.double() - b).abs().max()) <= 1e-4 * float(b.abs().max())


def test_vgg_layout_is_torchvisions():
    tv = pytest.importorskip("torchvision")
    from neo360_b200.lpips import LPIPS
    want = {k: v.shape for k, v in tv.models.vgg16().state_dict().items() if k.startswith("features.")}
    assert want == {f"features.{k}": v.shape for k, v in LPIPS().features.state_dict().items()}


def test_from_files_rejects_bad_keys(tmp_path, vgg):
    from neo360_b200.lpips import LPIPS
    ws = lm.lin_weights(4)
    good_lin = lm.lin_state(ws, "lpips")
    cases = []
    sd = dict(vgg); del sd["features.12.bias"]; cases.append((sd, good_lin, "features.12.bias"))
    sd = dict(vgg); sd["features.5.weight"] = sd["features.5.weight"][:, :3]; cases.append((sd, good_lin, "features.5.weight"))
    sd = dict(vgg); sd["features.31.weight"] = torch.zeros(1); cases.append((sd, good_lin, "features.31.weight"))
    lin = dict(good_lin); del lin["lin3.model.1.weight"]; cases.append((vgg, lin, "lin3.model.1.weight"))
    lin = lm.lin_state(ws, "piqa"); lin["2.1.weight"] = lin["2.1.weight"][:, :10]; cases.append((vgg, lin, "2.1.weight"))
    for i, (sd, lin, key) in enumerate(cases):
        torch.save(sd, tmp_path / f"v{i}.pth")
        torch.save(lin, tmp_path / f"l{i}.pth")
        with pytest.raises((KeyError, ValueError), match=key.replace(".", r"\.")):
            LPIPS.from_files(str(tmp_path / f"v{i}.pth"), str(tmp_path / f"l{i}.pth"))


@pytest.mark.parametrize("x,y", [(0, 0), (0, 130), (70, 0), (70, 130)])
def test_patch_order_at_the_corners(x, y):
    from neo360_b200 import batches
    T, H, W, view = 3, 100, 160, 2
    got = batches.patch_pix_inds(view, x, y, H, W)
    ref = torch.arange(T * H * W).view(T, H, W)[view].view(H, W)[x:x + 30, y:y + 30].reshape(-1)
    assert torch.equal(got, ref)
    with pytest.raises(ValueError):
        batches.patch_pix_inds(view, x + 1 if x else -1, y, H, W)

