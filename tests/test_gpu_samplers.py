"""GPU: the two inverse-CDF resamplers held per sample to oracle/sampler_model.py.

* `neo_sample_pdf`, called as each caller calls it (NeO-360 fg with pts, bg with pts and pts_lin, vanilla NeRF with far = pts = NULL):
  t equal to the fp32 emulation of `resample_kernel` bit for bit; every new sample admissible against the float64 operation
  (eps = (2 ceil(nw/32) + 16) 2^-24 a priori, delta = 4 ulp); the old values present bit for bit and the output sorted (descending for
  bg); fg pts and pts_lin bit for bit; bg pts within BG_PTS of float64 `depth2pts_outside` at the kernel's own s.  n_old in
  {4, 5, 33, ..., 257}, m in {1, 6, ..., 256}, n in {1, 3, 4, 5, 37, 4097}, one case near the 200 KB shared-memory limit; every batch
  mixes the weight families of tests/test_sampler_model.py; u deterministic, random, and exactly 0, 1 and on the emulated fp32 knots
  and one ulp either side.
* `neo_mip_resample`, levels 0 / 1 / 2: level 0 exactly (its cdf is [0, 1], so sdist shows the kernel's u formula); levels 1 / 2 every
  sdist within the interval that the float64 centre sandwiches give it and tdist within TDIST_K 2^-24 of float64 s_to_t of the kernel's
  own sdist; at train_frac = 0, rays with a NaN logit (0 * log 0) follow the reference's own sample_intervals.

Run with `-m gpu -s` to see the measured fraction of each bound.
"""
import numpy as np
import pytest
import torch

from oracle import mip_oracle as mor
from oracle import neo360_oracle as orc
from oracle import sampler_model as sm

pytestmark = pytest.mark.gpu

BG_PTS = 2e-5          # bg pts (asinf / sinf / cosf) vs float64 depth2pts_outside at the kernel's s
TDIST_K = 8.0          # tdist relative error / 2^-24 against float64 s_to_t of the kernel's sdist
N_OLD = [4, 5, 33, 34, 35, 36, 65, 66, 129, 130, 257]
M = [1, 6, 31, 32, 33, 64, 128, 256]
FAMILIES = sm.FAMILIES
WORST = {}


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


def note(key, v):
    WORST[key] = max(WORST.get(key, 0.0), float(v))


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    print("\nmeasured (largest over all cases): " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(WORST.items())))


def batch(n, n_old, rng):
    """Rays from inside the unit sphere, t ascending in [0.004, 2.5] (bg uses t / 2.5 descending), one weight family per ray."""
    t = np.empty((n, n_old), np.float32)
    w = np.empty((n, n_old), np.float32)
    for i in range(n):
        t[i:i + 1], w[i:i + 1] = sm.weight_family(FAMILIES[i % len(FAMILIES)], 1, n_old, rng)
    t = (t / np.float32(6.01) * np.float32(2.5)).astype(np.float32)
    o = rng.standard_normal((n, 3))
    o = (o / np.linalg.norm(o, axis=-1, keepdims=True) * 0.8 * rng.random((n, 1))).astype(np.float32)   # inside the unit sphere
    d = rng.standard_normal((n, 3)).astype(np.float32)
    d = (d / np.linalg.norm(d, axis=-1, keepdims=True)).astype(np.float32)
    return t, w, o, d


def u_set(mode, t, w, m, rng):
    n = t.shape[0]
    if mode == "det":
        return None
    u = rng.random((n, m)).astype(np.float32)
    if mode == "edges":
        _, cdf = sm.neo_cdf32(t, w)
        knots = np.concatenate([cdf, np.nextafter(cdf, np.float32(2)), np.nextafter(cdf, np.float32(-1)),
                                np.zeros((n, 1), np.float32), np.ones((n, 1), np.float32)], -1)
        knots = np.clip(knots, 0, 1).astype(np.float32)
        pick = rng.integers(0, knots.shape[1], (n, m))
        u = np.take_along_axis(knots, pick, -1)
        u[:, 0], u[:, -1] = 0.0, 1.0
    return np.ascontiguousarray(u)


def run_pdf(branch, t, w, o, d, m, u, dev):
    n, n_old = t.shape
    N1 = n_old + m
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    to, wo, oo, do = T(t), T(w), T(o), T(d)
    uu = T(u) if u is not None else None
    out = torch.full((n, N1), float("nan"), device=dev)
    pts = lin = None
    if branch == "fg":
        far = T(sm.ray_far32(o, d))
        pts = torch.full((n, N1, 3), float("nan"), device=dev)
        call("neo_sample_pdf", P(oo), P(do), P(far), P(to), P(wo), n, n_old, m, 1, 3.0, P(uu), P(out), P(pts), None)
    elif branch == "bg":
        far = T(sm.ray_far32(o, d))
        pts = torch.full((n, N1, 4), float("nan"), device=dev)
        lin = torch.full((n, N1, 3), float("nan"), device=dev)
        call("neo_sample_pdf", P(oo), P(do), P(far), P(to), P(wo), n, n_old, m, 0, 3.0, P(uu), P(out), P(pts), P(lin))
    else:                                           # vanilla NeRF's fine level (vanilla.cu / vanilla.py): far = pts = NULL
        call("neo_sample_pdf", P(oo), P(do), None, P(to), P(wo), n, n_old, m, 1, 0.0, P(uu), P(out), None, None)
    torch.cuda.synchronize()
    return out.cpu().numpy(), None if pts is None else pts.cpu().numpy(), None if lin is None else lin.cpu().numpy()


def check_pdf(branch, t, w, o, d, m, u, dev):
    ins = 0 if branch == "bg" else 1
    tt = t if ins else (t[:, ::-1] / np.float32(2.5)).astype(np.float32)     # bg: s in [0, 1] descending, as sample_along_rays leaves it
    got, pts, lin = run_pdf(branch, tt, w, o, d, m, u, dev)
    emu = sm.neo_resample(tt, w, m, ins, u_rand=u, o=o, d=d, far_unc=3.0)
    bad = got.view(np.int32) != emu["t"].view(np.int32)
    if bad.any():
        i, j = np.argwhere(bad)[0]
        raise AssertionError(f"{branch} n_old={t.shape[1]} m={m}: {int(bad.sum())} t differ from the emulation, first ray {i} slot {j}: "
                             f"kernel {got[i, j]!r} emulation {emu['t'][i, j]!r}")
    # sorted, and the old values present bit for bit
    assert (np.diff(got, axis=-1) >= 0).all() if ins else (np.diff(got, axis=-1) <= 0).all()
    merged = np.sort(np.concatenate([tt, emu["new"]], -1), -1)
    assert np.array_equal(np.sort(got, -1).view(np.int32), merged.view(np.int32))
    frac = sm.neo_admissible(tt, w, emu["new"], emu["u"], ins)
    note(f"{branch} eps fraction", frac.max())
    assert frac.max() <= 1.0, (branch, t.shape[1], m, frac.max())
    if branch == "fg":
        assert np.array_equal(pts.view(np.int32), emu["pts"].view(np.int32))
    if branch == "bg":
        assert np.array_equal(lin.view(np.int32), emu["pts_lin"].view(np.int32))
        assert np.array_equal(pts[..., 3].view(np.int32), got.view(np.int32))
        ref = orc.depth2pts_outside(torch.from_numpy(o).double(), torch.from_numpy(d).double(), torch.from_numpy(got).double())
        e = float(np.abs(pts[..., :3] - ref[..., :3].numpy()).max())
        note("bg pts", e)
        assert e <= BG_PTS, e


@pytest.mark.parametrize("n_old", N_OLD)
def test_sample_pdf_per_sample(cuda, n_old):
    rng = np.random.default_rng(n_old)
    for m in M:
        for branch in ("fg", "bg", "vanilla"):
            for mode in ("det", "rand", "edges"):
                t, w, o, d = batch(37, n_old, rng)
                check_pdf(branch, t, w, o, d, m, u_set(mode, t, w, m, rng), cuda)


@pytest.mark.parametrize("n,n_old,m", [(1, 4, 1), (3, 5, 6), (4, 33, 31), (5, 66, 64), (4097, 65, 64), (4097, 129, 64),
                                       (4097, 257, 128), (9, 1025, 7000)])
def test_sample_pdf_ray_counts_and_largest(cuda, n, n_old, m):
    """Ray counts that are not a multiple of the 4 warps per block, the configs' 64+1 / 128+1 / 256+1, and 1025 + 7000 samples
    (4 warps x (4 K + P2) floats, P2 = 8192: 192 KB of the 200 KB the launcher allows)."""
    rng = np.random.default_rng(n + n_old)
    for branch in ("fg", "bg", "vanilla"):
        for mode in ("det", "rand", "edges"):
            t, w, o, d = batch(n, n_old, rng)
            check_pdf(branch, t, w, o, d, m, u_set(mode, t, w, m, rng), cuda)


# ------------------------------------------------------------------------------------------------ Mip-NeRF 360

N_PREV = [1, 2, 31, 32, 33, 64, 160]
N_NEW = [2, 3, 31, 32, 33, 64, 160]


def mip_run(s_prev, w_prev, n, n_prev, level, N, near, far, train_frac, jitter, dev):
    T = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    sp, wp, j = T(s_prev), T(w_prev), T(jitter)          # kept alive until the kernel has run
    s = torch.empty(n, N + 1, device=dev)
    t = torch.empty(n, N + 1, device=dev)
    call("neo_mip_resample", P(sp), P(wp), n, n_prev, level, N, near, far, train_frac, P(j), P(s), P(t))
    torch.cuda.synchronize()
    return s.cpu().numpy(), t.cpu().numpy()


def mip_batch(n, n_prev, rng):
    """Per ray one of: rand**4, zero-weight runs, one-hot, points piled at 0 / 1 (the dilation clips: empty intervals, -inf logits)."""
    s = np.sort(rng.random((n, n_prev + 1)), -1).astype(np.float32)
    s[:, 0], s[:, -1] = 0.0, 1.0
    w = (rng.random((n, n_prev)) ** 4).astype(np.float32)
    kind = np.arange(n) % 4
    L = max(1, n_prev // 4)
    zr = kind == 1
    w[zr, :L] = 0.0
    w[zr, -L:] = 0.0
    w[zr] = np.where(rng.random((int(zr.sum()), n_prev)) < 0.3, 0.0, w[zr])
    oh = kind == 2
    w[oh] = 0.0
    w[np.nonzero(oh)[0], rng.integers(0, n_prev, int(oh.sum()))] = 1.0
    pile = kind == 3
    k = max(1, (n_prev + 1) // 4)
    s[pile, :k] = 0.0
    s[pile, -k:] = 1.0
    w = (w / np.maximum(w.sum(-1, keepdims=True), 1e-30)).astype(np.float32)
    return s, w


def jitters(mode, n, rng):
    if mode is None:
        return None
    j = rng.random(n).astype(np.float32)
    j[0::3] = 0.0
    j[1::3] = 1 - 2 ** -24
    return j


@pytest.mark.parametrize("near,far", [(0.2, 6.0), (0.2, 100.0)])
@pytest.mark.parametrize("n_new", N_NEW)
def test_mip_resample_level0_exact(cuda, n_new, near, far):
    rng = np.random.default_rng(n_new)
    for mode in (None, "mix"):
        j = jitters(mode, 37, rng)
        s, t = mip_run(None, None, 37, 1, 0, n_new, near, far, 0.5, j, cuda)
        assert any(np.array_equal(s.view(np.int32), c.view(np.int32)) for c in sm.mip_level0_sdist(37, n_new, j)), (n_new, mode)
        rel = np.abs(t - 1.0 / (s.astype(np.float64) / far + (1.0 - s.astype(np.float64)) / near)) * (
            s.astype(np.float64) / far + (1.0 - s.astype(np.float64)) / near) / sm.U
        note("mip tdist 2^-24", rel.max())
        assert rel.max() <= TDIST_K


@pytest.mark.parametrize("level", [1, 2])
@pytest.mark.parametrize("n_prev", N_PREV)
def test_mip_resample_per_sample(cuda, level, n_prev):
    rng = np.random.default_rng(10 * n_prev + level)
    for n_new in N_NEW:
        for train_frac in (0.0, 0.5, 1.0):
            for mode, (near, far) in ((None, (0.2, 6.0)), ("mix", (0.2, 100.0))):
                n = 37
                sp, wp = mip_batch(n, n_prev, rng)
                j = jitters(mode, n, rng)
                s, t = mip_run(sp, wp, n, n_prev, level, n_new, near, far, train_frac, j, cuda)
                td, wd = sm.mip_dilate(sp, wp, level)
                an = sm.mip_anneal(train_frac)
                c = sm.mip_check(td, wd, an, n_new, s, t, near, far, j)
                ok = ~c["collapse"]
                frac = c["sdist"][ok].max(initial=0.0)
                note("mip sdist offset from its interval middle (1 = at an end)", frac)
                note("mip tdist 2^-24", c["tdist"].max())
                assert frac <= 1.0, (level, n_prev, n_new, train_frac, mode, frac)
                assert c["tdist"].max() <= TDIST_K
                if c["collapse"].any():
                    ref = reference_sdist(td, wd, an, n_new, j)
                    cl = c["collapse"]
                    assert np.array_equal(s[cl], ref[cl]), (level, n_prev, n_new, train_frac, s[cl][0], ref[cl][0])


def reference_sdist(td, wd, anneal, n_new, jitter=None):
    td_t, wd_t = torch.tensor(td), torch.tensor(wd)
    lg = torch.where(td_t[:, 1:] > td_t[:, :-1], torch.tensor(anneal) * torch.log(wd_t + 0.0), torch.full_like(wd_t, -torch.inf))
    j = None if jitter is None else torch.tensor(jitter)[:, None]
    return mor.sample_intervals(td_t, lg, n_new, j).numpy()


def test_mip_resample_nan_logit_follows_the_reference(cuda):
    """train_frac = 0 (anneal 0): a non-empty interval whose dilated weight is exactly 0 gets the reference logit 0 * log 0 = NaN;
    the reference's softmax, cumsum and sorted_interp then put every centre on the first knot, so sdist is the first knot throughout."""
    sp = np.array([[0.0, 0.1, 0.2, 0.5, 0.7, 0.8, 1.0]], np.float32)
    wp = np.array([[0.3, 0.0, 0.0, 0.0, 0.5, 0.2]], np.float32)
    td, wd = sm.mip_dilate(sp, wp, 1)
    assert ((wd == 0) & (td[:, 1:] > td[:, :-1])).any()
    for j in (None, np.array([0.5], np.float32)):
        s, _ = mip_run(sp, wp, 1, 6, 1, 8, 0.2, 6.0, 0.0, j, cuda)
        ref = reference_sdist(td, wd, sm.mip_anneal(0.0), 8, j)
        assert np.array_equal(ref, np.full_like(ref, td[0, 0]))
        assert np.array_equal(s, ref), (s, ref)
