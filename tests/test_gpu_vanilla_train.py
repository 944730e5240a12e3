"""GPU: the training path of vanilla NeRF (`NeRF.forward` under autograd, neo360_b200/vanilla.py).

* `neo_vanilla_composite_bwd` (composite_bwd_kernel in mode 2) and the mode-2 forward against the float64 model
  (oracle/vanilla_train_model.py, pinned to autograd through `vanilla_oracle.composite` by tests/test_vanilla_train_model.py):
  N in {1, 2, 31, 32, 33, 64, 65, 129, 193, 257}, n in {1, 127, 128, 129, 4096}, white and black, |rays_d| from 0.3 to 3, t from the
  library's own samplers at 65 / 129 / 193; every batch mixes transparent rays, one opaque sample, runs of opaque samples (T underflows),
  an opaque first sample, all-zero sigma, duplicate t and a tiny sigma on the 1e10 interval; each upstream gradient alone, then all.
  Units as tests/test_gpu_train_stages.py: forward |got - model| in 2^-24 N (depth relative to max t), backward in 2^-24 N magnitude.
* `neo_vanilla_sample_along_rays` / `neo_sample_pdf` give the eval path's t bit for bit; `neo_vanilla_encode` gives the fp32 point
  bit for bit and sin columns within a few fp32 ulp of float64 sin of the kernel's own argument; the training path's per-sample sigma / rgb
  equal the fused fp32 eval field kernel's to GEMM re-association.
* end to end: the training tuples equal `vanilla_oracle.render` and the fp32 eval forward; gradients of the reference loss (MSE of both
  levels) and of a loss that also uses acc and depth equal autograd through the oracle's MLP and compositing at the library's sample
  positions (which carry no gradient: the reference detaches the level-0 weights).
* eval after one Adam step (fp32 and tc) uses the updated weights.

Bounds are 2-3x the largest values measured on an H100 80GB HBM3 at a 400 W power limit (DESIGN.md section 2).  Run with `-m gpu -s`
to see the measured values.
"""
import pytest
import torch

from neo360_b200 import synth
from oracle import neo360_oracle as orc
from oracle import vanilla_oracle as vo
from oracle import vanilla_train_model as vtm

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
DENORM = 2.0 ** -126
OUT_ROUND = 2.0 ** -149
COMP_FWD_K = 4.0          # measured 1.52
COMP_BWD_K = 8.0          # measured 3.39 (at N = 1), mean 0.0094
ENC_SIN_ABS = 4 * 2.0 ** -24   # sinf is within 2 ulp (<= 2^-23 for |sin| <= 1)
FIELD_K = 6e-6            # per-sample sigma (relative to max(1, max sigma)) / rgb, training GEMMs vs the fused eval kernel: measured 2.4e-6
TUPLE_EVAL_K = 2.5e-5     # training tuples vs the fp32 eval forward: measured 9.5e-6
COMP_N = [1, 2, 31, 32, 33, 64, 65, 129, 193, 257]
COMP_RAYS = [1, 127, 128, 129, 4096]
NEAR, FAR = 2.0, 6.0


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


def sample(o, vd, nc, u0=None, near=NEAR, far=FAR):
    t = torch.empty(o.shape[0], nc + 1, device=o.device)
    call("neo_vanilla_sample_along_rays", P(o), P(vd), o.shape[0], nc, near, far, P(u0), P(t))
    return t


def resample(o, vd, t0, w0, nf, u1=None):
    t = torch.empty(o.shape[0], t0.shape[1] + nf, device=o.device)
    call("neo_sample_pdf", P(o), P(vd), None, P(t0), P(w0), o.shape[0], t0.shape[1], nf, 1, 0.0, P(u1), P(t), None, None)
    return t


# ---------------------------------------------------------------- compositing stage

def comp_inputs(n, N, seed, dev):
    g = torch.Generator(device=dev).manual_seed(seed)
    vd = torch.nn.functional.normalize(torch.randn(n, 3, generator=g, device=dev), dim=-1)
    o = torch.randn(n, 3, generator=g, device=dev)
    d = vd * (0.3 + 2.7 * torch.rand(n, 1, generator=g, device=dev))                  # |rays_d| != 1 (quirk Q15)
    if N in (65, 129, 193):
        t = sample(o, vd, 64 if N == 65 else 128, torch.rand(n, 129 if N != 65 else 65, generator=g, device=dev))
        if N == 193:
            t = resample(o, vd, t, torch.rand(n, 129, generator=g, device=dev) ** 4, 64, torch.rand(n, 64, generator=g, device=dev))
    else:
        t = NEAR + (FAR - NEAR) * torch.sort(torch.rand(n, N, generator=g, device=dev), -1)[0]
    reg = (torch.arange(n, device=dev) + seed) % 8
    t = t.clone()
    dup = (reg == 5).nonzero()[:, 0]
    if N > 1:
        j = torch.arange(1, N, 3, device=dev)
        t[dup[:, None], j[None]] = t[dup[:, None], (j - 1)[None]]
    t64 = t.double()
    dist = torch.cat([t64[:, 1:] - t64[:, :-1], torch.full_like(t64[:, :1], 1e10)], 1) * d.double().norm(dim=-1, keepdim=True)
    sig = torch.nn.functional.softplus(torch.randn(n, N, generator=g, device=dev, dtype=torch.float64) * 2 - 1)
    sig[reg == 0] *= 1e-3                                                            # transparent
    sig[reg == 4] = 0.0                                                              # all-zero sigma
    sig[reg == 6, N - 1] = 1e-12                                                     # tiny sigma on the 1e10 interval
    vals = torch.tensor([17.0, 18.0, 30.0, 1e3], device=dev, dtype=torch.float64)
    rows = torch.arange(n, device=dev)
    k1 = torch.randint(0, N, (n,), generator=g, device=dev)
    ok = dist > 1e-6

    def opaque(mask, col, v):
        m = mask & ok[rows, col]
        sig[rows[m], col[m]] = (v / dist[rows, col])[m]

    opaque(reg == 2, k1, vals[rows % 4])                                             # one opaque sample
    opaque(reg == 7, torch.zeros_like(k1), vals[rows % 4])                           # opaque first sample
    if N >= 6:                                                                       # runs of 5..8 opaque samples
        k0 = torch.randint(0, max(1, N - 8), (n,), generator=g, device=dev)
        for r in range(8):
            opaque((reg == 3) & (r < 5 + rows % 4), (k0 + r).clamp(max=N - 1), 18.0 + 3 * r)
    rgb = torch.rand(n, N, 3, generator=g, device=dev)
    ups = {"g_comp": torch.randn(n, 3, generator=g, device=dev), "g_acc": torch.randn(n, generator=g, device=dev),
           "g_w": torch.randn(n, N, generator=g, device=dev), "g_depth": torch.randn(n, generator=g, device=dev)}
    return rgb.contiguous(), sig.float().contiguous(), t.contiguous(), d.contiguous(), ups


def comp_fwd(rgb, sig, t, d, white):
    n, N = t.shape
    out = dict(comp=torch.empty(n, 3, device=t.device), acc=torch.empty(n, device=t.device), w=torch.empty(n, N, device=t.device),
               depth=torch.empty(n, device=t.device))
    call("neo_volumetric_rendering", P(rgb), P(sig), P(t), P(d), None, n, N, int(white), 2, P(out["comp"]), P(out["acc"]), P(out["w"]),
         None, P(out["depth"]))
    return out


def comp_bwd(rgb, sig, t, d, white, gs):
    n, N = t.shape
    d_rgb = torch.full((n, N, 3), float("nan"), device=t.device)
    d_sig = torch.full((n, N), float("nan"), device=t.device)
    call("neo_vanilla_composite_bwd", P(rgb), P(sig), P(t), P(d), n, N, int(white), *[P(gs.get(k)) for k in ("g_comp", "g_acc", "g_w", "g_depth")],
         P(d_rgb), P(d_sig))
    return d_rgb, d_sig


def bwd_ratio(d_rgb, d_sig, m, gs, N):
    """|got - model| in units of 2^-24 N (magnitude + subnormal floor), after the absolute rounding of a subnormal fp32 output (the units
    of tests/test_gpu_train_stages.py)."""
    gmax = m["G_mag"].amax(1)[:, None]
    floor_s = DENORM * gmax / m["a"] * m["dist"] * m["e"]
    es = ((d_sig.double() - m["d_sigma"]).abs() - OUT_ROUND).clamp_min(0)
    rs = es / (U * N * (m["d_sigma_mag"] + floor_s)).clamp_min(1e-300)
    gc = gs["g_comp"].double().abs()[:, None, :] if "g_comp" in gs else torch.zeros_like(m["d_rgb"])
    er = ((d_rgb.double() - m["d_rgb"]).abs() - OUT_ROUND / 2 * (gc + 1)).clamp_min(0)
    rr = er / (U * N * (m["d_rgb_mag"] + DENORM * gc)).clamp_min(1e-300)
    rs = torch.where(torch.isnan(d_sig), torch.full_like(rs, float("inf")), rs)
    rr = torch.where(torch.isnan(d_rgb), torch.full_like(rr, float("inf")), rr)
    return torch.cat([rs.reshape(-1), rr.reshape(-1)])


@pytest.mark.parametrize("white", [True, False], ids=["white", "black"])
def test_vanilla_composite_backward_vs_float64(cuda, white):
    names = ["g_comp", "g_acc", "g_w", "g_depth"]
    worst_f, worst_b, means_b, where_b = 0.0, 0.0, [], None
    for N in COMP_N:
        for n in COMP_RAYS:
            rgb, sig, t, d, ups = comp_inputs(n, N, 1000 * N + n + 3 * white, cuda)
            got = comp_fwd(rgb, sig, t, d, white)
            mf = vtm.composite_fwd(rgb, sig, t, d, white)
            tmax = t.double().abs().amax(1)
            rf = torch.stack([(got["comp"].double() - mf["comp"]).abs().amax(1), (got["acc"].double() - mf["acc"]).abs(),
                              (got["w"].double() - mf["w"]).abs().amax(1), (got["depth"].double() - mf["depth"]).abs() / tmax], 1) / (U * N)
            worst_f = max(worst_f, float(rf.max()))
            for use in [[k] for k in names] + [names]:
                gs = {k: ups[k] for k in use}
                d_rgb, d_sig = comp_bwd(rgb, sig, t, d, white, gs)
                rb = bwd_ratio(d_rgb, d_sig, vtm.composite_bwd(rgb, sig, t, d, white, **gs), gs, N)
                if float(rb.max()) > worst_b:
                    worst_b, where_b = float(rb.max()), (N, n, use)
                means_b.append(float(rb.mean()))
    tag = f"vanilla composite {'white' if white else 'black'}"
    print(f"{tag} forward: max {worst_f:.3g} x 2^-24 N (bound {COMP_FWD_K})")
    print(f"{tag} backward: max {worst_b:.3g} at (N, n, upstream) {where_b}, mean {sum(means_b) / len(means_b):.3g} x 2^-24 N magnitude "
          f"(bound {COMP_BWD_K})")
    assert worst_f <= COMP_FWD_K and worst_b <= COMP_BWD_K, (worst_f, worst_b, where_b)


def test_composite_autograd_wrapper_mode_2(cuda):
    """training._Composite in mode 2: the kernels behind autograd, every output used; bg_lambda is zeros."""
    from neo360_b200.training import _Composite
    rgb, sig, t, d, ups = comp_inputs(129, 65, 5, cuda)
    r, s = rgb.clone().requires_grad_(True), sig[..., None].clone().requires_grad_(True)
    comp, acc, w, lam, depth = _Composite.apply(r, s, t, d, None, True, 2)
    assert bool((lam == 0).all())
    loss = (comp * ups["g_comp"]).sum() + (acc * ups["g_acc"]).sum() + (w * ups["g_w"]).sum() + (depth * ups["g_depth"]).sum()
    loss.backward()
    rb = bwd_ratio(r.grad, s.grad[..., 0], vtm.composite_bwd(rgb, sig, t, d, True, **ups), ups, 65)
    print(f"_Composite mode 2: max {float(rb.max()):.3g}")
    assert float(rb.max()) <= COMP_BWD_K


# ---------------------------------------------------------------- sampling and encodings

def frame(n, seed, dev, scale=True):
    """n rays of a 32 x 24 view of the turntable; rays_d scaled to |rays_d| in [0.5, 2] (viewdirs stay unit)."""
    W, H = 32, 24
    ro, vd, rd, _ = orc.rays_from_pose(orc.ray_directions(H, W, 0.8 * W), synth.target_pose(5 + seed, 100)[:3, :4])
    sel = torch.arange(100, 100 + n) % ro.shape[0]
    g = torch.Generator().manual_seed(seed)
    s = 0.5 + 1.5 * torch.rand(n, 1, generator=g) if scale else torch.ones(n, 1)
    return {"rays_o": ro[sel].contiguous(), "rays_d": (rd[sel] * s).contiguous(), "viewdirs": vd[sel].contiguous()}


NEAR_V, FAR_V = 0.2, 3.0       # the near / far of the vanilla parity tests (tests/test_gpu_parity.py)


def uniforms(n, nc, nf, seed):
    g = torch.Generator().manual_seed(100 + seed)
    return [torch.rand(n, nc + 1, generator=g), torch.rand(n, nf, generator=g)]


@pytest.mark.parametrize("nc,nf", [(8, 4), (64, 64)])
def test_vanilla_sampling_and_encodings_match_eval(cuda, nc, nf):
    from neo360_b200 import vanilla
    from neo360_b200.vanilla import NeRF
    n = 96
    rays = {k: v.to(cuda) for k, v in frame(n, 1, cuda).items()}
    u = [x.to(cuda) for x in uniforms(n, nc, nf, 1)]
    net = NeRF(num_coarse_samples=nc, num_fine_samples=nf).eval()
    net.load_state_dict(synth.make_vanilla_params(1))
    net = net.to(cuda)
    o, vd = rays["rays_o"], rays["viewdirs"]
    for randomized in (False, True):
        with torch.no_grad():
            net(dict(rays, _uniforms=u), randomized, False, NEAR_V, FAR_V, debug=True)
        dbg = net.last_debug
        t0 = sample(o, vd, nc, u[0] if randomized else None, NEAR_V, FAR_V)
        assert torch.equal(t0, dbg["t"][0])
        t1 = resample(o, vd, t0, dbg["weights"][0], nf, u[1] if randomized else None)
        assert torch.equal(t1, dbg["t"][1])
        for lvl, (t, mlp) in enumerate(((t0, net.coarse_mlp), (t1, net.fine_mlp))):
            N = t.shape[1]
            enc, denc = torch.empty(n * N, 63, device=cuda), torch.empty(n, 27, device=cuda)
            call("neo_vanilla_encode", P(o), P(vd), P(t), n, N, P(enc), P(denc))
            pts = o[:, None, :] + t[..., None] * vd[:, None, :]                       # fp32 mul, then fp32 add: the kernel's point
            assert torch.equal(enc[:, :3], pts.reshape(-1, 3)) and torch.equal(denc[:, :3], vd)
            for e, x, deg in ((enc, pts.reshape(-1, 3), 10), (denc, vd, 4)):
                xb = (x[:, None, :] * torch.tensor([2.0 ** k for k in range(deg)], device=cuda)[:, None]).reshape(x.shape[0], -1)
                arg = torch.cat([xb, xb + 1.5707963705062866], -1)                 # fp32 adds, as the kernel's add_
                err = (e[:, 3:].double() - torch.sin(arg.double())).abs()
                print(f"encoding sin / cos columns vs float64 sin of the kernel's argument: {float(err.max()):.2e}")
                assert float(err.max()) <= ENC_SIN_ABS, float(err.max())
            with torch.no_grad():
                raw_rgb, raw_sigma = vanilla._mlp_train(mlp, enc, denc, n, N)
                sig = torch.nn.functional.softplus(raw_sigma - 1.0)[..., 0]
                rgb = torch.sigmoid(raw_rgb) * 1.002 - 0.001
            es, er = float((sig - dbg["sigma"][lvl].reshape(n, N)).abs().max()), float((rgb - dbg["rgb_s"][lvl]).abs().max())
            print(f"nc+nf {nc}+{nf} level {lvl} randomized {randomized}: training GEMMs vs fused eval kernel sigma {es:.2e} rgb {er:.2e}")
            assert es <= FIELD_K * max(1.0, float(dbg["sigma"][lvl].abs().max())) and er <= FIELD_K, (es, er)


# ---------------------------------------------------------------- end to end

def oracle_train(rays, Pg, nc, nf, white, ts):
    """vanilla_oracle.render's MLP and compositing under autograd at the sample positions `ts` (one (n, N_l) tensor per level) of the
    training call.  The positions carry no gradient (the reference detaches the level-0 weights, helper.py:613); taking the training
    call's own keeps an inverse-CDF sample that lands in a neighbouring bin (a cdf value within rounding of its uniform: level-0 weights
    from other GEMMs, or from the oracle) from counting as a gradient error.  The samplers are checked separately: bit-identical to the
    eval path on the same weights (test_vanilla_sampling_and_encodings_match_eval), which tests/test_gpu_parity.py holds to the reference."""
    o, d, vd = rays["rays_o"], rays["rays_d"], rays["viewdirs"]
    denc = orc.pos_enc(vd, 0, 4)
    ret = []
    for lvl, t in enumerate(ts):
        pts = o[:, None, :] + t[..., None] * vd[:, None, :]
        raw_rgb, raw_sigma = vo.mlp_forward(Pg, "coarse_mlp." if lvl == 0 else "fine_mlp.", orc.pos_enc(pts, 0, 10), denc)
        rgb = torch.sigmoid(raw_rgb) * (1 + 2 * 0.001) - 0.001
        sigma = torch.nn.functional.softplus(raw_sigma - 1.0)
        comp, acc, w, depth = vo.composite(rgb, sigma, t, d, white)
        ret.append((comp, acc, depth))
    return ret


def losses(ret, target):
    mse = ((ret[0][0] - target) ** 2).mean() + ((ret[1][0] - target) ** 2).mean()        # LitNeRF.training_step, model.py:273-299
    full = mse + sum((lv[1] ** 2).mean() + 0.1 * lv[2].mean() for lv in ret)
    return {"mse": mse, "mse+acc+depth": full}


def md(a, b):
    return float((a.detach().cpu().double() - b.detach().cpu().double()).abs().max())


@pytest.mark.parametrize("white", [True, False], ids=["white", "black"])
@pytest.mark.parametrize("nc,nf", [(8, 4), (64, 64)])
def test_vanilla_training_forward_and_gradients_vs_oracle(cuda, nc, nf, white):
    """Stated: tuples 2e-4 against the oracle (fp32 CPU); against the fp32 eval forward TUPLE_EVAL_K; every parameter's gradient within
    1e-2 of its gradient scale in max norm and 3e-3 in relative L2 (the bounds of tests/test_training.py)."""
    from neo360_b200.vanilla import NeRF
    n, seed = 24, nc + white
    rays = frame(n, seed, cuda)
    u = uniforms(n, nc, nf, seed)
    Pm = synth.make_vanilla_params(seed)
    target = torch.rand(n, 3, generator=torch.Generator().manual_seed(9))
    drays = {k: v.to(cuda) for k, v in rays.items()}
    du = [x.to(cuda) for x in u]
    net = NeRF(num_coarse_samples=nc, num_fine_samples=nf)
    net.load_state_dict(Pm)
    net = net.to(cuda).train()
    with torch.no_grad():
        ref_fwd = vo.render(rays, Pm, nc, nf, NEAR_V, FAR_V, white, rand={"u0": u[0], "u1": u[1]})
        ev = net.eval()(dict(drays, _uniforms=du), True, white, NEAR_V, FAR_V)
    net.train()
    rel2 = lambda a, b: float((a.detach().cpu().double() - b.detach().cpu().double()).norm() / max(float(b.detach().cpu().double().norm()), 1e-30))
    for name in ("mse", "mse+acc+depth"):
        net.zero_grad(set_to_none=True)
        got = net(dict(drays, _uniforms=du), True, white, NEAR_V, FAR_V, debug=True)
        assert got[1][0].requires_grad
        Pg = {k: v.clone().requires_grad_(True) for k, v in Pm.items()}
        ref = oracle_train(rays, Pg, nc, nf, white, [t.cpu() for t in net.last_debug["t"]])
        losses(ref, target)[name].backward()
        e_ref = max(md(a, b) for lv in range(2) for a, b in zip(got[lv], ref_fwd[lv]))
        e_ev = max(md(a, b) for lv in range(2) for a, b in zip(got[lv], ev[lv]))
        assert e_ref < 2e-4 and e_ev < TUPLE_EVAL_K, (e_ref, e_ev)
        losses(got, target.to(cuda))[name].backward()
        worst, worst2 = 0.0, 0.0
        for pname, p in net.named_parameters():
            gref = Pg[pname].grad
            scale = float(gref.abs().max())
            err, e2 = md(p.grad, gref), rel2(p.grad, gref)
            worst, worst2 = max(worst, err / max(scale, 1e-12)), max(worst2, e2)
            assert err < 1e-2 * scale + 1e-9 and e2 < 3e-3, (name, pname, err, scale, e2)
        print(f"{nc}+{nf} {'white' if white else 'black'} [{name}]: tuples vs oracle {e_ref:.2e}, vs fp32 eval {e_ev:.2e}; "
              f"worst gradient max-abs / scale {worst:.2e}, relative L2 {worst2:.2e}")


def test_vanilla_eval_after_a_training_step_uses_the_new_weights(cuda):
    """Eval (fp32 and tc) before a step packs the weights; one Adam step changes them in place; the next eval call must re-pack and
    reproduce the oracle with the UPDATED weights (fp32 2e-4, tc 3e-2: the bounds of tests/test_gpu_parity.py) and differ from the old."""
    from neo360_b200.vanilla import NeRF
    nc, nf, n = 16, 8, 64
    rays = frame(n, 3, cuda)
    drays = {k: v.to(cuda) for k, v in rays.items()}
    Pm = synth.make_vanilla_params(3)
    net = NeRF(num_coarse_samples=nc, num_fine_samples=nf)
    net.load_state_dict(Pm)
    net = net.to(cuda)
    before = {}
    for prec in ("fp32", "tc"):
        net.precision = prec
        with torch.no_grad():
            before[prec] = net.eval()(drays, False, True, NEAR_V, FAR_V)[1][0]
    net.train()
    opt = torch.optim.Adam(net.parameters(), lr=5e-4)     # the reference's lr_init
    target = torch.rand(n, 3, generator=torch.Generator().manual_seed(4)).to(cuda)
    losses(net(drays, True, True, NEAR_V, FAR_V), target)["mse"].backward()
    opt.step()
    P2 = {k: v.detach().cpu() for k, v in net.state_dict().items()}
    ref_new = vo.render(rays, P2, nc, nf, NEAR_V, FAR_V, True)[1][0]
    ref_old = vo.render(rays, Pm, nc, nf, NEAR_V, FAR_V, True)[1][0]
    assert md(ref_new, ref_old) > 1e-3
    for prec, tol in (("fp32", 2e-4), ("tc", 3e-2)):
        net.precision = prec
        with torch.no_grad():
            got = net.eval()(drays, False, True, NEAR_V, FAR_V)[1][0]
        print(f"eval {prec} after a step: vs new weights {md(got, ref_new):.2e}, vs old {md(got, ref_old):.2e}, moved {md(got, before[prec]):.2e}")
        assert md(got, ref_new) < tol and md(got, before[prec]) > 1e-3 and md(got, ref_new) < md(got, ref_old), prec
