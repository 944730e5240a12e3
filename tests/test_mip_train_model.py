"""CPU: the Mip-NeRF 360 training path without a GPU.

* The float64 model of `neo_mip_composite_bwd` (oracle/mip_train_model.py) with its roundings off equals torch.autograd through
  `mip_oracle`'s head activations + `alpha_weights` + white-background rendering, values and gradients, to 1e-12 of its magnitude unit.
* `mip.training_loss` (searchsorted / cumsum / gather form of lossfun_outer, O(N) distortion) equals the reference's mask / O(N^2) forms
  (`mip_train_oracle.lossfun_outer`, `lossfun_distortion`) in float64, values and gradients, with tied and domain-clipped sdist.
* `mip._mlp_train` (direction columns of views_linear.0 applied once per ray) equals `mip_oracle.mlp` in float64.
* `mip_train_oracle` reproduces the reference's training loss and gradients pinned in tests/golden/mip360_train_vectors.npz.
* The new entry points reject bad arguments before any launch (the pointers are never dereferenced).
"""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import mip_oracle as mor
from oracle import mip_train_oracle as mto
from oracle import mip_train_model as mtm

GRADS = ("g_rgb", "g_w", "g_density", "g_rgb_s")
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "mip360_train_vectors.npz")


def composite_case(N, seed, n=12):
    """Ascending tdist with non-unit |d| (0.3 .. 3): realistic raw density, an opaque run, an opaque first sample, very negative raw density
    (transparent), raw density above the softplus threshold, saturated raw rgb, duplicate t."""
    g = torch.Generator().manual_seed(seed)
    t = 0.2 + 6.0 * torch.sort(torch.rand(n, N + 1, generator=g, dtype=torch.float64), -1)[0]
    r = torch.randn(n, N, generator=g, dtype=torch.float64) * 2
    if N >= 8:
        r[1, 1:7] = 40.0
        t[4, 2:5] = t[4, 1]
    r[2, 0] = 60.0
    r[3] = -30.0
    r[5] = 25.0
    q = torch.randn(n, N, 3, generator=g, dtype=torch.float64) * 3
    q[6] = 40.0
    q[7] = -40.0
    d = torch.randn(n, 3, generator=g, dtype=torch.float64)
    d = d / d.norm(dim=-1, keepdim=True) * (0.3 + 2.7 * torch.rand(n, 1, generator=g, dtype=torch.float64))
    ups = {"g_rgb": torch.randn(n, 3, generator=g, dtype=torch.float64), "g_w": torch.randn(n, N, generator=g, dtype=torch.float64),
           "g_density": torch.randn(n, N, generator=g, dtype=torch.float64), "g_rgb_s": torch.randn(n, N, 3, generator=g, dtype=torch.float64)}
    return r, q, t, d, ups


def oracle_stage(r, q, t, d):
    """The reference's stage through mip_oracle: activations (model.py:142-173), alpha_weights, rendering with bg 1 (helper.py:264-274)."""
    density = F.softplus(r - 1.0)
    rgb = torch.sigmoid(q) * (1 + 2 * 0.001) - 0.001 if q is not None else torch.zeros(*r.shape, 3, dtype=r.dtype)
    w = mor.alpha_weights(density, t, d)
    acc = w.sum(-1)
    out = (w[..., None] * rgb).sum(-2) + torch.clip(1 - acc[..., None], min=0) * 1.0
    return {"g_rgb": out, "g_w": w, "g_density": density, "g_rgb_s": rgb}


@pytest.mark.parametrize("N", [1, 2, 9, 33, 40])
@pytest.mark.parametrize("nerf", [True, False], ids=["nerf", "proposal"])
def test_mip_composite_model_equals_autograd(N, nerf):
    """Every upstream gradient alone and all together; N = 1 is the infinite interval alone; rays whose float64 acc lands either side of 1."""
    r, q, t, d, ups = composite_case(N, 7 * N + nerf)
    if not nerf:
        q = None
    ms = set()
    for use in [[k] for k in GRADS] + [list(GRADS)]:
        if not nerf and use == ["g_rgb_s"]:
            continue
        rl = r.clone().requires_grad_(True)
        ql = q.clone().requires_grad_(True) if nerf else None
        outs = oracle_stage(rl, ql, t, d)
        loss = sum((outs[k] * ups[k]).sum() for k in use if nerf or k != "g_rgb_s")
        gr = torch.autograd.grad(loss, [rl] + ([ql] if nerf else []), allow_unused=True, materialize_grads=True)
        m = mtm.composite_bwd(r, q, t, d, fp32=False, **{k: ups[k] for k in use})
        ms.update(m["m"].tolist())
        pairs = [(m["d_raw_density"], gr[0], m["d_raw_density_mag"])] + ([(m["d_raw_rgb"], gr[1], m["d_raw_rgb_mag"])] if nerf else [])
        for got, ref, mag in pairs:
            err = (got - ref).abs()
            assert bool((err <= 1e-12 * mag + 1e-300).all()), (use, float((err / mag.clamp_min(1e-300)).max()))
    f = mtm.composite_fwd(r, q, t, d, fp32=False)
    o = oracle_stage(r, q, t, d)
    for a, b in ((f["rgb"], o["g_rgb"]), (f["w"], o["g_w"]), (f["density"], o["g_density"]), (f["rgb_s"], o["g_rgb_s"])):
        assert float((a - b).abs().max()) <= 1e-13 * max(1.0, float(b.abs().max()))
    if N >= 9:
        assert ms == {0.0, 1.0}, ms           # the clip's gradient both passed and blocked among these rays


def test_mip_composite_model_rounds_like_the_kernel():
    """fp32 on: delta is the fp32 product fp32(t_{k+1} - t_k) * fp32 |d|, x = fp32(fp32 density * delta), the exclusive scan in fp32 in
    the kernel's warp order; fp32 off: float64."""
    g = torch.Generator().manual_seed(3)
    n, N = 3, 70
    t = torch.sort(torch.rand(n, N + 1, generator=g, dtype=torch.float64), -1)[0] * 5 + 0.2
    r = torch.randn(n, N, generator=g, dtype=torch.float64)
    d = torch.randn(n, 3, generator=g, dtype=torch.float64)
    k32, k64 = mtm.composite_terms(r, t, d, fp32=True), mtm.composite_terms(r, t, d, fp32=False)
    d32, t32 = d.float(), t.float()
    dn = torch.sqrt((d32[:, 0] * d32[:, 0] + d32[:, 1] * d32[:, 1]) + d32[:, 2] * d32[:, 2])
    assert torch.equal(k32["delta"], ((t32[:, 1:] - t32[:, :-1]) * dn[:, None]).double())
    x32 = (F.softplus((r.float() - 1.0).double()).float().double() * k32["delta"]).float()
    assert torch.equal(k32["x"][:, :-1], x32[:, :-1].double()) and bool(torch.isinf(k32["x"][:, -1]).all())
    # the warp scan: sequential float32 sums differ from it, the float64 sum is within N ulp of it
    assert float((k32["excl"] - k64["excl"]).abs().max()) < N * 2.0 ** -23 * float(k64["excl"].abs().max())
    v = x32[:, :32].clone()                    # the carry into the second chunk: lane 31's Hillis-Steele sum of x_0 .. x_31
    for o in (1, 2, 4, 8, 16):
        v = torch.cat([v[:, :o], v[:, o:] + v[:, :-o]], 1)
    assert torch.equal(k32["excl"][:, 32], v[:, 31].double())


# ---------------------------------------------------------------- losses

def loss_case(seed, n=10, Np=(12, 12), Nn=8):
    g = torch.Generator().manual_seed(seed)

    def sd(N):
        s = torch.sort(torch.rand(n, N + 1, generator=g, dtype=torch.float64), -1)[0]
        s[0, :3] = 0.0                                   # clipped to the domain start
        s[1, -3:] = 1.0                                  # clipped to the domain end
        s[2, 4:7] = s[2, 4]                              # ties
        return s
    hist = []
    for N in (*Np, Nn):
        w = torch.rand(n, N, generator=g, dtype=torch.float64)
        w = (w / w.sum(-1, keepdim=True)).requires_grad_(True)
        hist.append({"sdist": sd(N), "weights": w})
    if Np[0] >= Nn:
        hist[-1]["sdist"][3] = hist[0]["sdist"][3, :Nn + 1]   # NeRF-level sdist equal to proposal sdist: ties across levels
    rgb = torch.rand(n, 3, generator=g, dtype=torch.float64).requires_grad_(True)
    target = torch.rand(n, 3, generator=g, dtype=torch.float64)
    return [{"rgb": rgb}], hist, target


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_training_loss_equals_the_reference_mask_forms(seed):
    from neo360_b200.mip import training_loss
    ren, hist, target = loss_case(seed, Np=(12, 20) if seed == 2 else (12, 12), Nn=8 if seed else 16)
    leaves = [ren[0]["rgb"]] + [h["weights"] for h in hist]
    data, inter, dist = mto.training_loss_terms(ren, hist, target)
    ref = data + inter + 0.01 * dist
    g_ref = torch.autograd.grad(ref, leaves)
    got = training_loss(ren, hist, target)
    g_got = torch.autograd.grad(got, leaves)
    assert abs(float(got) - float(ref)) <= 1e-12 * max(1.0, abs(float(ref)))
    for a, b in zip(g_got, g_ref):
        assert float((a - b).abs().max()) <= 1e-12 * max(1.0, float(b.abs().max()))
    # the searchsorted form gives the mask form's brackets exactly
    from neo360_b200.mip import _outer_weights
    c = hist[-1]["sdist"]
    for h in hist[:-1]:
        lo, hi = mto.searchsorted(h["sdist"], c)
        r = torch.searchsorted(h["sdist"].contiguous(), c.contiguous(), right=True)
        assert torch.equal(lo, (r - 1).clamp(min=0)) and torch.equal(hi, r.clamp(max=h["sdist"].shape[-1] - 1))
        cy = torch.cat([torch.zeros_like(h["weights"][..., :1]), torch.cumsum(h["weights"], -1)], -1)
        want = torch.take_along_dim(cy, hi, -1)[..., 1:] - torch.take_along_dim(cy, lo, -1)[..., :-1]
        assert torch.equal(_outer_weights(c, h["sdist"], h["weights"]), want)


# ---------------------------------------------------------------- MLP and golden

def test_training_mlp_equals_the_oracle_mlp_in_float64():
    from neo360_b200 import synth
    from neo360_b200.mip import MipNeRF360, _mlp_train
    P = {k: v.double() for k, v in synth.make_mip_params(2, width=64).items()}
    net = MipNeRF360(num_prop_samples=8, num_nerf_samples=4).double()
    net.mlps[2] = type(net.mlps[2])(netwidth=64).double()
    net.load_state_dict(P)
    g = torch.Generator().manual_seed(0)
    n, N = 3, 5
    feats, vd = torch.randn(n * N, 504, generator=g, dtype=torch.float64), F.normalize(torch.randn(n, 3, generator=g, dtype=torch.float64), dim=-1)
    denc = mor.dir_enc(vd)
    for lvl in range(3):
        Pg = {k: v.clone().requires_grad_(True) for k, v in P.items()}
        dens_r, rgb_r = mor.mlp(Pg, f"mlps.{lvl}.", feats.reshape(n, N, 504), vd, 4 if lvl < 2 else 8, lvl < 2)
        net.zero_grad(set_to_none=True)
        rd, rc = _mlp_train(net.mlps[lvl], feats, denc, n, N)
        dens = F.softplus(rd - 1.0)
        assert float((dens - dens_r).detach().abs().max()) < 1e-12
        loss_r, loss = dens_r.sin().sum(), dens.sin().sum()
        if lvl == 2:
            rgb = torch.sigmoid(rc) * 1.002 - 0.001
            assert float((rgb - rgb_r).detach().abs().max()) < 1e-12
            loss_r, loss = loss_r + rgb_r.cos().sum(), loss + rgb.cos().sum()
        else:
            assert rc is None
        loss_r.backward()
        loss.backward()
        for name, p in net.mlps[lvl].named_parameters():
            ref = Pg[f"mlps.{lvl}.{name}"].grad
            assert float((p.grad - ref).abs().max()) <= 1e-12 * max(1.0, float(ref.abs().max())), (lvl, name)


@pytest.mark.parametrize("tag", ["t_tiny", "t_small"])
def test_oracle_reproduces_the_reference_training_step(tag):
    """mip_train_oracle's loss terms and per-parameter gradient norms / projections equal the reference's pinned values."""
    from neo360_b200 import synth
    from oracle.make_golden_mip_train import oracle_step, probes
    z = np.load(GOLDEN)
    W, H, B, npp, nn_, seed = (int(v) for v in z[f"{tag}_cfg"])
    batch = {k: torch.from_numpy(z[f"{tag}_{k}"]) for k in ("rays_o", "rays_d", "viewdirs", "radii")}
    jit = [torch.from_numpy(z[f"{tag}_jit{i}"]) for i in range(3)]
    (data, inter, dist), g = oracle_step(batch, synth.make_mip_params(seed), npp, nn_, jit, torch.from_numpy(z[f"{tag}_target"]))
    loss = torch.stack([data, inter, dist]).detach().double()
    assert float((loss - torch.from_numpy(z[f"{tag}_loss"]).double()).abs().max()) < 1e-5
    names = [str(s) for s in z[f"{tag}_names"]]
    r = probes([(k, g[k]) for k in names], seed)
    gn, gd = torch.from_numpy(z[f"{tag}_gnorm"]), torch.from_numpy(z[f"{tag}_gdot"])
    for i, k in enumerate(names):
        gk = g[k].double()
        assert abs(float(gk.norm()) - float(gn[i])) <= 1e-3 * float(gn[i]) + 1e-12, k
        assert abs(float((gk * r[k]).sum()) - float(gd[i])) <= 1e-3 * float(gn[i]) * float(r[k].norm()) + 1e-12, k


# ---------------------------------------------------------------- argument checks

@pytest.fixture(scope="module")
def lib():
    from neo360_b200 import build, _lib
    build.build()
    return _lib.load()


def test_mip_training_entry_points_validate_arguments_without_gpu(lib):
    from neo360_b200 import _lib as L
    for name in ("neo_mip_resample", "neo_mip_encode", "neo_mip_composite", "neo_mip_composite_bwd"):
        assert name in L.SYMBOLS and hasattr(lib, name)
    p = 1 << 20
    rs = lambda sp, wp, n, npv, lvl, nn, s, t, near=0.2, far=6.0: lib.neo_mip_resample(sp, wp, n, npv, lvl, nn, near, far, 0.5, None, s, t, None)
    for args in ((p, p, 4, 8, 3, 8, p, p), (p, p, 4, 8, -1, 8, p, p), (None, p, 4, 8, 1, 8, p, p), (p, None, 4, 8, 2, 8, p, p),
                 (p, p, 4, 8, 1, 8, None, p), (p, p, 4, 8, 1, 8, p, None), (p, p, 0, 8, 1, 8, p, p), (p, p, -2, 8, 1, 8, p, p),
                 (p, p, 4, 0, 1, 8, p, p), (p, p, 4, 8, 1, 1, p, p), (p, p, 4, 8, 1, 161, p, p), (None, None, 4, 1, 0, 8, p, p, 0.0),
                 (None, None, 4, 1, 0, 8, p, p, 2.0, 1.0)):
        assert rs(*args) == -1, args
    assert b"neo_mip_resample" in lib.neo_last_error()
    enc = lambda *a: lib.neo_mip_encode(*a, None)
    base = [p, p, p, p, p, p, 4, 8, p, p]
    for i in list(range(6)) + [8, 9]:
        a = list(base)
        a[i] = None
        assert enc(*a) == -1, i
    for i, v in ((6, 0), (6, -1), (7, 0)):
        a = list(base)
        a[i] = v
        assert enc(*a) == -1, (i, v)
    assert b"neo_mip_encode" in lib.neo_last_error()
    comp = lambda rd, rc, t, d, n, N: lib.neo_mip_composite(rd, rc, t, d, n, N, p, p, p, p, None)
    for args in ((None, p, p, p, 4, 8), (p, p, None, p, 4, 8), (p, p, p, None, 4, 8), (p, p, p, p, 0, 8), (p, p, p, p, 4, 0)):
        assert comp(*args) == -1, args
    assert b"neo_mip_composite" in lib.neo_last_error()
    bwd = lambda rd, rc, t, d, n, N, dd, dc: lib.neo_mip_composite_bwd(rd, rc, t, d, n, N, p, None, None, None, dd, dc, None)
    for args in ((None, p, p, p, 4, 8, p, p), (p, p, None, p, 4, 8, p, p), (p, p, p, None, 4, 8, p, p), (p, p, p, p, 4, 8, None, p),
                 (p, p, p, p, 4, 8, p, None), (p, p, p, p, 0, 8, p, p), (p, p, p, p, -1, 8, p, p), (p, p, p, p, 4, 0, p, p),
                 (p, None, p, p, 4, 8, None, None)):
        assert bwd(*args) == -1, args
    assert b"neo_mip_composite_bwd" in lib.neo_last_error()
