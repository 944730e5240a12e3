"""GPU: the training path of Mip-NeRF 360 (`MipNeRF360.forward` under autograd, neo360_b200/mip.py).

* `neo_mip_composite_bwd` and the forward `neo_mip_composite` (the eval path's composite_kernel) against the float64 model
  (oracle/mip_train_model.py, pinned to autograd through `mip_oracle` by tests/test_mip_train_model.py): n in {1, 127, 128, 129, 4096},
  N in {1, 2, 31, 32, 33, 64, 65, 160}, tdist from `neo_mip_resample` at levels 0 / 1 / 2 or sorted random with duplicates; every batch
  mixes transparent rays, opaque runs (T underflows), zero density, raw density above the softplus threshold and saturated rgb; proposal
  (raw rgb NULL) and NeRF levels; each upstream gradient alone, then all.  Forward in 2^-24 N absolute (density 2^-24 relative), backward
  in 2^-24 N of the model's magnitude unit.
* `neo_mip_resample`, fed the eval path's own history, gives the eval path's next-level sdist bit for bit (deterministic and jittered).
* `neo_mip_encode`: at level 0 (whose sdist depends on no weights) the training path's density / rgb equal the fp32 eval forward's history
  to GEMM re-association; the features equal float64 `mip_oracle` features of the same tdist within a measured bound.
* end to end: training renderings vs the fp32 eval forward at the same jitter (level 0 within a bound; levels 1 and 2 for >= 99 % of rays,
  because resampling on other weights can move a sample across a bracket); gradients of `training_loss`, and of a loss that also uses the
  ray_history density / rgb and the proposal renderings, w.r.t. every parameter of the three MLPs against autograd through the float64 oracle
  at the training call's own sdist.

Bounds are 2-3x the largest values measured on an H100 80GB HBM3 at a 700 W power limit (DESIGN.md section 2).  Run with `-m gpu -s` to
see the measured values.
"""
import pytest
import torch
import torch.nn.functional as F

from neo360_b200 import synth
from neo360_b200.mip_basis import POS_BASIS_T
from oracle import mip_oracle as mor
from oracle import mip_train_model as mtm
from oracle import neo360_oracle as orc

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
DENORM = 2.0 ** -126
OUT_ROUND = 2.0 ** -149
COMP_FWD_K = 6.0           # forward |got - model| / (2^-24 N): measured 2.47
COMP_DENS_K = 8.0          # activated density, relative / 2^-24: measured 3.97
COMP_BWD_K = 12.0          # backward |got - model| / (2^-24 N magnitude): measured 5.56 (NeRF level, N = 1), 2.81 (proposal)
FEAT_ABS = 2e-4            # IPE features vs float64 mip_oracle at the same tdist: measured 7.3e-5
FIELD_K = 5e-7             # level-0 density (relative to max(1, max density)) / NeRF-level rgb, training GEMMs vs the eval SGEMM chain: measured 1.8e-7
REN_K = 4e-7               # training renderings vs the fp32 eval forward: measured 1.2e-7 (level 0), 1.8e-7 (levels 1, 2)
COMP_N = [1, 2, 31, 32, 33, 64, 65, 160]
COMP_RAYS = [1, 127, 128, 129, 4096]
NEAR, FAR = 0.2, 6.0


@pytest.fixture(scope="module")
def cuda():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from neo360_b200 import build
    build.build()
    return torch.device("cuda:0")


def call(name, *args):
    from neo360_b200 import _lib as L
    L.check(getattr(L.load(), name)(*args, torch.cuda.current_stream().cuda_stream))


def P(t):
    from neo360_b200 import _lib as L
    return L.ptr(t)


def resample(s_prev, w_prev, n, n_prev, level, N, jitter=None, train_frac=0.5, near=NEAR, far=FAR, dev=None):
    s = torch.empty(n, N + 1, device=dev)
    t = torch.empty(n, N + 1, device=dev)
    call("neo_mip_resample", P(s_prev), P(w_prev), n, n_prev, level, N, near, far, train_frac, P(jitter), P(s), P(t))
    return s, t


# ---------------------------------------------------------------- compositing stage

def comp_inputs(n, N, seed, dev):
    g = torch.Generator(device=dev).manual_seed(seed)
    vd = F.normalize(torch.randn(n, 3, generator=g, device=dev), dim=-1)
    d = vd * (0.3 + 2.7 * torch.rand(n, 1, generator=g, device=dev))
    src = seed % 4 if N >= 2 else 3
    if src < 3:                                   # tdist of the library's resampling at level `src`
        lvl = src
        n_prev = 1 if lvl == 0 else max(2, N // 2)
        sp = torch.sort(torch.rand(n, n_prev + 1, generator=g, device=dev), -1)[0]
        sp[:, 0], sp[:, -1] = 0.0, 1.0
        wp = torch.rand(n, n_prev, generator=g, device=dev) ** 4
        wp = (wp / wp.sum(-1, keepdim=True)).contiguous()
        _, t = resample(sp.contiguous(), wp, n, n_prev, lvl, N, torch.rand(n, generator=g, device=dev), dev=dev)
    else:                                         # sorted random with duplicates
        t = NEAR + (FAR - NEAR) * torch.sort(torch.rand(n, N + 1, generator=g, device=dev), -1)[0]
    reg = (torch.arange(n, device=dev) + seed) % 8
    t = t.clone()
    dup = (reg == 5).nonzero()[:, 0]
    if N > 1:
        j = torch.arange(1, N + 1, 3, device=dev)
        t[dup[:, None], j[None]] = t[dup[:, None], (j - 1)[None]]
    r = torch.randn(n, N, generator=g, device=dev) * 2
    r[reg == 0] = -12.0 + r[reg == 0]                                          # transparent
    r[reg == 1] = -200.0                                                       # zero density (softplus underflows)
    r[reg == 2] = 21.0 + 10 * torch.rand_like(r[reg == 2])                     # above the softplus threshold
    if N >= 6:                                                                 # runs of opaque samples: T underflows behind them
        k0 = torch.randint(0, max(1, N - 8), (n,), generator=g, device=dev)
        rows = (reg == 3).nonzero()[:, 0]
        for i in range(6):
            r[rows, (k0[rows] + i).clamp(max=N - 1)] = 60.0 + 20 * i
    r[reg == 7, 0] = 80.0                                                      # opaque first sample
    q = torch.randn(n, N, 3, generator=g, device=dev) * 2
    q[reg == 6] = 40.0 * torch.sign(q[reg == 6])                               # saturated rgb
    ups = {"g_rgb": torch.randn(n, 3, generator=g, device=dev), "g_w": torch.randn(n, N, generator=g, device=dev),
           "g_density": torch.randn(n, N, generator=g, device=dev), "g_rgb_s": torch.randn(n, N, 3, generator=g, device=dev)}
    return r.contiguous(), q.contiguous(), t.contiguous(), d.contiguous(), ups


def comp_fwd(r, q, t, d):
    n, N = r.shape
    out = dict(rgb=torch.empty(n, 3, device=r.device), w=torch.empty(n, N, device=r.device), density=torch.empty(n, N, device=r.device),
               rgb_s=torch.full((n, N, 3), float("nan"), device=r.device))
    call("neo_mip_composite", P(r), P(q), P(t), P(d), n, N, P(out["rgb"]), P(out["w"]), P(out["density"]), P(out["rgb_s"]))
    return out


def comp_bwd(r, q, t, d, gs):
    n, N = r.shape
    d_r = torch.full((n, N), float("nan"), device=r.device)
    d_q = torch.full((n, N, 3), float("nan"), device=r.device) if q is not None else None
    call("neo_mip_composite_bwd", P(r), P(q), P(t), P(d), n, N, *[P(gs.get(k)) for k in ("g_rgb", "g_w", "g_density", "g_rgb_s")], P(d_r), P(d_q))
    return d_r, d_q


def bwd_ratio(d_r, d_q, m, gs, N):
    """|got - model| in units of 2^-24 N magnitude, after the absolute rounding of a subnormal fp32 output; a subnormal floor for products
    that underflow inside the kernel."""
    gmax = sum(gs[k].double().abs().amax(tuple(range(1, gs[k].dim()))) for k in gs)[:, None]
    es = ((d_r.double() - m["d_raw_density"]).abs() - OUT_ROUND).clamp_min(0)
    rs = es / (U * N * (m["d_raw_density_mag"] + DENORM * (1 + gmax))).clamp_min(1e-300)
    rs = torch.where(torch.isnan(d_r), torch.full_like(rs, float("inf")), rs)
    if d_q is None:
        return rs.reshape(-1)
    er = ((d_q.double() - m["d_raw_rgb"]).abs() - OUT_ROUND).clamp_min(0)
    rr = er / (U * N * (m["d_raw_rgb_mag"] + DENORM * (1 + gmax[..., None]))).clamp_min(1e-300)
    rr = torch.where(torch.isnan(d_q), torch.full_like(rr, float("inf")), rr)
    return torch.cat([rs.reshape(-1), rr.reshape(-1)])


@pytest.mark.parametrize("nerf", [True, False], ids=["nerf", "proposal"])
def test_mip_composite_stage_vs_float64(cuda, nerf):
    names = ["g_rgb", "g_w", "g_density", "g_rgb_s"] if nerf else ["g_rgb", "g_w", "g_density"]
    worst_f, worst_d, worst_b, where_b, means_b = 0.0, 0.0, 0.0, None, []
    for N in COMP_N:
        for n in COMP_RAYS:
            r, q, t, d, ups = comp_inputs(n, N, 1000 * N + n + nerf, cuda)
            qq = q if nerf else None
            got = comp_fwd(r, qq, t, d)
            mf = mtm.composite_fwd(r, qq, t, d)
            rf = torch.stack([(got["rgb"].double() - mf["rgb"]).abs().amax(1), (got["w"].double() - mf["w"]).abs().amax(1),
                              (got["rgb_s"].double() - mf["rgb_s"]).abs().amax((1, 2))], 1) / (U * N)
            rd = ((got["density"].double() - mf["density"]).abs() - OUT_ROUND).clamp_min(0) / (U * mf["density"]).clamp_min(1e-300)
            worst_f, worst_d = max(worst_f, float(rf.max())), max(worst_d, float(rd.max()))
            for use in [[k] for k in names] + [names]:
                gs = {k: ups[k] for k in use}
                d_r, d_q = comp_bwd(r, qq, t, d, gs)
                rb = bwd_ratio(d_r, d_q, mtm.composite_bwd(r, qq, t, d, **gs), gs, N)
                if float(rb.max()) > worst_b:
                    worst_b, where_b = float(rb.max()), (N, n, use)
                means_b.append(float(rb.mean()))
    tag = "mip composite " + ("nerf" if nerf else "proposal")
    print(f"{tag} forward: max {worst_f:.3g} x 2^-24 N (bound {COMP_FWD_K}), density {worst_d:.3g} x 2^-24 relative (bound {COMP_DENS_K})")
    print(f"{tag} backward: max {worst_b:.3g} at (N, n, upstream) {where_b}, mean {sum(means_b) / len(means_b):.3g} x 2^-24 N magnitude "
          f"(bound {COMP_BWD_K})")
    assert worst_f <= COMP_FWD_K and worst_d <= COMP_DENS_K and worst_b <= COMP_BWD_K, (worst_f, worst_d, worst_b, where_b)


# ---------------------------------------------------------------- resampling and encoding

def mip_rays(n, seed, W=64, H=48):
    """n rays of a 64 x 48 turntable target view (reference get_rays arithmetic via the oracle), |rays_d| != 1, radii of the pixel cone."""
    ro, vd, rd, radii = orc.rays_from_pose(orc.ray_directions(H, W, 0.8 * W), synth.target_pose(9 + seed, 100)[:3, :4])
    sel = torch.randperm(H * W, generator=torch.Generator().manual_seed(seed))[:n]
    return {"rays_o": ro[sel].contiguous(), "rays_d": rd[sel].contiguous(), "viewdirs": vd[sel].contiguous(),
            "radii": radii[sel].reshape(-1, 1).contiguous()}


def make_net(npp, nn_, seed, dev):
    from neo360_b200.mip import MipNeRF360
    net = MipNeRF360(num_prop_samples=npp, num_nerf_samples=nn_)
    net.load_state_dict(synth.make_mip_params(seed))
    return net.to(dev)


@pytest.mark.parametrize("npp,nn_", [(16, 8), (64, 32)])
def test_resample_and_encode_match_eval(cuda, npp, nn_):
    n = 128
    rays = {k: v.to(cuda) for k, v in mip_rays(n, 1).items()}
    net = make_net(npp, nn_, 1, cuda).eval()
    jit = [torch.rand(n, 1, generator=torch.Generator().manual_seed(5 + i)).to(cuda) for i in range(3)]
    ns = (npp, npp, nn_)
    for randomized in (False, True):
        with torch.no_grad():
            ren, hist = net(dict(rays, _uniforms=jit), 0.5, randomized, True, NEAR, FAR)
        for lvl in range(3):
            sp = hist[lvl - 1]["sdist"].contiguous() if lvl else None
            wp = hist[lvl - 1]["weights"].contiguous() if lvl else None
            s, t = resample(sp, wp, n, ns[lvl - 1] if lvl else 1, lvl, ns[lvl], jit[lvl].reshape(-1).contiguous() if randomized else None, dev=cuda)
            assert torch.equal(s, hist[lvl]["sdist"]), (randomized, lvl)
        # level 0: features vs float64 oracle at the same tdist; training GEMMs vs the eval SGEMM chain
        s0 = hist[0]["sdist"]
        t0 = 1 / (s0 * (1 / FAR) + (1 - s0) * (1 / NEAR))
        _, t0k = resample(None, None, n, 1, 0, npp, jit[0].reshape(-1).contiguous() if randomized else None, dev=cuda)
        feats, denc = torch.empty(n * npp, 504, device=cuda), torch.empty(n, 27, device=cuda)
        basis = net.mlps[0].pos_basis_t.contiguous()
        call("neo_mip_encode", P(rays["rays_o"]), P(rays["rays_d"]), P(rays["viewdirs"]), P(rays["radii"].reshape(-1).contiguous()), P(t0k), P(basis),
             n, npp, P(feats), P(denc))
        b64 = {k: v.double() for k, v in rays.items()}
        mean, cov = mor.cast_cone(t0k.double(), b64["rays_o"], b64["rays_d"], b64["radii"])
        ref = mor.ipe_features(*mor.contract(mean, cov), basis.double()).reshape(n * npp, 504)
        ef = float((feats.double() - ref).abs().max())
        ed = float((denc.double() - mor.dir_enc(b64["viewdirs"])).abs().max())
        from neo360_b200.mip import _mlp_train
        with torch.no_grad():
            rd, _ = _mlp_train(net.mlps[0], feats, denc, n, npp)
            dens = F.softplus(rd - 1.0)
        edn = float((dens - hist[0]["density"]).abs().max()) / max(1.0, float(hist[0]["density"].abs().max()))
        print(f"{npp}/{nn_} randomized {randomized}: features vs float64 {ef:.2e}, dir enc {ed:.2e}, level-0 density training vs eval {edn:.2e} "
              f"(tdist of the eval path vs s_to_t: {float((t0k - t0).abs().max()):.1e})")
        assert ef <= FEAT_ABS and ed <= FEAT_ABS and edn <= FIELD_K, (ef, ed, edn)
        # the NeRF level's rgb through the same encoding of its tdist
        s2 = hist[2]["sdist"]
        s2k, t2 = resample(hist[1]["sdist"].contiguous(), hist[1]["weights"].contiguous(), n, npp, 2, nn_,
                           jit[2].reshape(-1).contiguous() if randomized else None, dev=cuda)
        assert torch.equal(s2k, s2)
        f2 = torch.empty(n * nn_, 504, device=cuda)
        call("neo_mip_encode", P(rays["rays_o"]), P(rays["rays_d"]), P(rays["viewdirs"]), P(rays["radii"].reshape(-1).contiguous()), P(t2),
             P(net.mlps[2].pos_basis_t.contiguous()), n, nn_, P(f2), P(denc))
        with torch.no_grad():
            rd2, rc2 = _mlp_train(net.mlps[2], f2, denc, n, nn_)
            rgb2 = torch.sigmoid(rc2) * 1.002 - 0.001
        er = float((rgb2 - hist[2]["rgb"]).abs().max())
        print(f"  NeRF-level rgb training GEMMs vs eval: {er:.2e}")
        assert er <= FIELD_K, er


# ---------------------------------------------------------------- end to end

def oracle_train(batch, Pg, sdists, target):
    """mip_oracle's MLPs and compositing under autograd in float64 at the sample positions `sdists` of the training call (they carry no
    gradient: stop_level_grad, model.py:309-310); returns (renderings, history) and the reference loss terms."""
    o, d, vd, radii = batch["rays_o"], batch["rays_d"], batch["viewdirs"], batch["radii"]
    ren, hist = [], []
    for lvl, s in enumerate(sdists):
        t = 1 / (s * (1 / FAR) + (1 - s) * (1 / NEAR))
        feats = mor.ipe_features(*mor.contract(*mor.cast_cone(t, o, d, radii)), POS_BASIS_T.to(o))
        density, rgb = mor.mlp(Pg, f"mlps.{lvl}.", feats, vd, 4 if lvl < 2 else 8, lvl < 2)
        w = mor.alpha_weights(density, t, d)
        acc = w.sum(-1)
        ren.append({"rgb": (w[..., None] * rgb).sum(-2) + torch.clip(1 - acc[..., None], min=0)})
        hist.append({"density": density, "rgb": rgb, "sdist": s, "weights": w})
    return ren, hist


def losses(ren, hist, target, name):
    from neo360_b200.mip import training_loss
    loss = training_loss(ren, hist, target)
    if name == "all outputs":
        loss = loss + sum(0.01 * h["density"].mean() + (h["rgb"] ** 2).mean() for h in hist) + sum(((r["rgb"] - target) ** 2).mean() for r in ren[:-1])
    return loss


@pytest.mark.parametrize("npp,nn_,n", [(16, 8, 256), (64, 32, 256)])
def test_mip_training_forward_and_gradients_vs_oracle(cuda, npp, nn_, n):
    seed = npp
    rays = {k: v.to(cuda) for k, v in mip_rays(n, seed).items()}
    jit = [torch.rand(n, 1, generator=torch.Generator().manual_seed(50 + i)).to(cuda) for i in range(3)]
    target = torch.rand(n, 3, generator=torch.Generator().manual_seed(9)).to(cuda)
    Pm = synth.make_mip_params(seed)
    net = make_net(npp, nn_, seed, cuda)
    with torch.no_grad():
        ev_ren, ev_hist = net.eval()(dict(rays, _uniforms=jit), 0.5, True, True, NEAR, FAR)
    net.train()
    b64 = {k: v.double() for k, v in rays.items()}
    rel2 = lambda a, b: float((a.double() - b.double()).norm() / max(float(b.double().norm()), 1e-30))
    for name in ("reference loss", "all outputs"):
        net.zero_grad(set_to_none=True)
        ren, hist = net(dict(rays, _uniforms=jit), 0.5, True, True, NEAR, FAR)
        assert ren[-1]["rgb"].requires_grad and hist[0]["weights"].requires_grad and not hist[2]["sdist"].requires_grad
        assert bool((hist[0]["rgb"] == 0).all()) and bool((hist[1]["rgb"] == 0).all())
        e0 = float((ren[0]["rgb"] - ev_ren[0]["rgb"]).detach().abs().max())
        err12 = [(ren[l]["rgb"] - ev_ren[l]["rgb"]).detach().abs().amax(-1) for l in (1, 2)]
        frac = [float((e <= REN_K).double().mean()) for e in err12]
        moved = [int((hist[l]["sdist"] != ev_hist[l]["sdist"]).any(-1).sum()) for l in (1, 2)]
        print(f"{npp}/{nn_} [{name}]: level 0 rendering vs fp32 eval {e0:.2e}; rays within {REN_K} at levels 1, 2: {frac} "
              f"(max {float(err12[0].max()):.2e}, {float(err12[1].max()):.2e}; rays whose sdist differs from eval: {moved})")
        assert e0 <= REN_K and min(frac) >= 0.99, (e0, frac)
        losses(ren, hist, target, name).backward()
        Pg = {k: v.to(cuda).double().requires_grad_(not k.endswith("pos_basis_t")) for k, v in Pm.items()}
        o_ren, o_hist = oracle_train(b64, Pg, [h["sdist"].double() for h in hist], target.double())
        losses(o_ren, o_hist, target.double(), name).backward()
        worst, worst2 = 0.0, 0.0
        for pname, p in net.named_parameters():
            gref = Pg[pname].grad
            scale = float(gref.abs().max())
            err, e2 = float((p.grad.double() - gref).abs().max()), rel2(p.grad, gref)
            worst, worst2 = max(worst, err / max(scale, 1e-12)), max(worst2, e2)
            assert err < 1e-2 * scale + 1e-9 and e2 < 3e-3, (name, pname, err, scale, e2)
        print(f"  gradients: worst max-abs / scale {worst:.2e}, relative L2 {worst2:.2e}")
