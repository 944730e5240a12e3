"""CPU: the models of the two inverse-CDF resamplers (oracle/sampler_model.py) and the argument checks of `neo_sample_pdf` /
`neo_sample_along_rays`.

* the float64 forms equal `neo360_oracle.piecewise_constant_pdf` / `resample_fg` / `resample_bg` / `vanilla_oracle.sample_pdf`
  in float64 to 1e-12 on every weight family of the GPU test;
* the fp32 emulation of `resample_kernel` is admissible against the float64 operation on >= 10^5 rays, so the bound is sound before
  any kernel is held to it;
* a catalogue of planted bugs, applied to the emulation, moves every mutant off the unmutated emulation bit for bit (the GPU bound)
  and, where the bug changes where the sample lands rather than which of two equal inverses it takes, outside the float64 bound;
* the Mip-NeRF 360 model: the fp32 stand-in passes its interval checks, its NaN-logit rays follow the reference form, and its two
  mutants leave the bounds.

Run with -s to see the measured fractions of each bound.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import mip_oracle as mor
from oracle import neo360_oracle as orc
from oracle import sampler_model as sm
from oracle import vanilla_oracle as vor

FAMILIES = sm.FAMILIES
weights = sm.weight_family
TOL = 1e-12


@pytest.mark.parametrize("fam", FAMILIES)
@pytest.mark.parametrize("n_old,m", [(5, 6), (34, 31), (65, 64)])
def test_float64_forms_equal_the_oracles(fam, n_old, m):
    rng = np.random.default_rng([FAMILIES.index(fam), n_old, m])
    n = 64
    t, w = weights(fam, n, n_old, rng)
    o = torch.randn(n, 3, dtype=torch.float64) * 0.1
    d = torch.nn.functional.normalize(torch.randn(n, 3, dtype=torch.float64), dim=-1)
    T, W = torch.tensor(t, dtype=torch.float64), torch.tensor(w, dtype=torch.float64)
    # the CPU oracle draws its deterministic u as torch's CPU fp32 linspace, which differs by an ulp from the CUDA one at some m
    u_det = torch.linspace(0.0, 1.0 - 2 ** -32, m).numpy()
    for u_rand, u_model in ((None, np.broadcast_to(u_det, (n, m))), (torch.rand(n, m, dtype=torch.float64),) * 2):
        um = np.asarray(u_model, np.float64)
        fg = sm.neo_resample(t.astype(np.float64), w.astype(np.float64), m, 1, u_rand=um, rounding=False)["t"]
        ref, _ = orc.resample_fg(o, d, T, W, m, u_rand)
        assert np.abs(fg - ref.numpy()).max() <= TOL
        ref, _ = vor.sample_pdf(o, d, T, W, m, u_rand)
        assert np.abs(fg - ref.numpy()).max() <= TOL
        S = torch.flip(T, [-1])
        bg = sm.neo_resample(S.numpy(), w.astype(np.float64), m, 0, u_rand=um, rounding=False)["t"]
        ref, _, _ = orc.resample_bg(o, d, S, W, m, torch.ones(n, 1, dtype=torch.float64), 3.0, u_rand)
        assert np.abs(bg - ref.numpy()).max() <= TOL


def test_fp32_emulation_is_admissible_on_1e5_rays():
    """The bound is sound: the emulation of the kernel's own fp32 arithmetic lies within eps (a priori) and delta of the float64
    operation, fg and bg, every family, random and deterministic u, >= 10^5 rays in all."""
    rng = np.random.default_rng(7)
    worst = {1: 0.0, 0: 0.0}
    rays = 0
    for n_old, m in ((5, 6), (36, 33), (66, 64), (130, 64)):
        for fam in FAMILIES:
            n = 900
            t, w = weights(fam, n, n_old, rng)
            u = rng.random((n, m)).astype(np.float32)
            u[: n // 4] = sm.linspace01(m)
            for ins in (1, 0):
                tt = t if ins else t[:, ::-1].copy()
                r = sm.neo_resample(tt, w, m, ins, u_rand=u)
                frac = sm.neo_admissible(tt, w, r["new"], r["u"], ins)
                assert frac.max() <= 1.0, (fam, n_old, m, ins, frac.max())
                worst[ins] = max(worst[ins], float(frac.max()))
                rays += n
    print(f"\nfp32 emulation vs float64, {rays} rays: largest fraction of eps needed fg {worst[1]:.3f}, bg {worst[0]:.3f}")
    assert rays >= 100_000


MUTANTS = {
    # name: (admissibility must fail as well, in which branches)
    "carry": (1, 0),            # carry dropped at the first block boundary
    "strict_search": (),        # `<` instead of `<=`: on flat runs it takes the other end of the same preimage
    "q17_neighbours": (0,),     # bins[lo] / bins[lo+1] instead of pmax / smin: only descending (bg) bins differ
    "pad_count": (1, 0),        # pad / (nw + 1)
    "w_shift": (1, 0),          # w[0:-2] instead of w[1:-1]
    "no_q7": (),                # the last u stays below 1: on a zero run at the end it lands on the run's other end
}


@pytest.mark.parametrize("mutant", sorted(MUTANTS))
def test_mutation_catalogue(mutant):
    rng = np.random.default_rng(11)
    diffs, worst = 0, {1: 0.0, 0: 0.0}
    for n_old, m in ((36, 33), (66, 64)):
        for fam in ("rand4", "zero_runs", "onehot_mid", "sum_below", "zero"):
            n = 64
            t, w = weights(fam, n, n_old, rng)
            u = np.broadcast_to(sm.linspace01(m), (n, m)).copy()
            # u exactly on the emulated knots makes the tie rule visible
            _, cdf = sm.neo_cdf32(t, w)
            u[:, : m // 2] = np.sort(cdf[:, 1:1 + m // 2], -1)
            for ins in (1, 0):
                tt = t if ins else t[:, ::-1].copy()
                ur = None if mutant == "no_q7" else u
                good = sm.neo_resample(tt, w, m, ins, u_rand=ur)
                bad = sm.neo_resample(tt, w, m, ins, u_rand=ur, mutate=mutant)
                diffs += int((good["t"].view(np.int32) != bad["t"].view(np.int32)).sum())
                worst[ins] = max(worst[ins], float(sm.neo_admissible(tt, w, bad["new"], good["u"], ins).max()))
    print(f"\n{mutant}: {diffs} samples off the emulation; largest fraction of the float64 bound fg {worst[1]:.3g}, bg {worst[0]:.3g}")
    assert diffs > 0
    for ins in MUTANTS[mutant]:
        assert worst[ins] > 1.0, (mutant, ins, worst)


# ------------------------------------------------------------------------------------------------ Mip-NeRF 360

def mip_inputs(n, n_prev, rng, kind):
    s = np.sort(rng.random((n, n_prev + 1)), -1).astype(np.float32)
    s[:, 0], s[:, -1] = 0.0, 1.0
    w = (rng.random((n, n_prev)) ** 4).astype(np.float32)
    if kind == "zero_runs":
        L = max(1, n_prev // 4)
        w[:, :L] = 0.0
        w[:, -L:] = 0.0
        w[rng.random((n, n_prev)) < 0.3] = 0.0
    elif kind == "onehot":
        w[:] = 0.0
        w[np.arange(n), rng.integers(0, n_prev, n)] = 1.0
    w = (w / np.maximum(w.sum(-1, keepdims=True), 1e-30)).astype(np.float32)
    return s, w


@pytest.mark.parametrize("level", [1, 2])
@pytest.mark.parametrize("train_frac", [0.0, 0.5, 1.0])
def test_mip_stand_in_within_bounds(level, train_frac):
    """The fp32 stand-in (np.log / np.exp for logf / expf) passes every interval check at levels 1 and 2; its NaN-logit rays give
    the reference's own outcome."""
    rng = np.random.default_rng(level * 10 + int(train_frac * 2))
    worst_s, worst_t = 0.0, 0.0
    for n_prev, n_new in ((2, 3), (33, 31), (64, 64), (160, 32)):
        for kind in ("rand4", "zero_runs", "onehot"):
            for jit in (None, "rand"):
                n = 96
                s, w = mip_inputs(n, n_prev, rng, kind)
                j = rng.random(n).astype(np.float32) if jit else None
                r = sm.mip_resample32(s, w, level, n_new, train_frac, 0.2, 6.0, j)
                c = sm.mip_check(r["td"], r["wd"], r["anneal"], n_new, r["sdist"], r["tdist"], 0.2, 6.0, j)
                ok = ~c["collapse"]
                assert c["sdist"][ok].max(initial=0) <= 1.0 and c["tdist"].max() <= 8.0
                worst_s, worst_t = max(worst_s, c["sdist"][ok].max(initial=0)), max(worst_t, c["tdist"].max())
                if c["collapse"].any():
                    ref = reference_sdist(r["td"], r["wd"], r["anneal"], n_new, j)
                    assert np.array_equal(r["sdist"][c["collapse"]], ref[c["collapse"]])
    print(f"\nmip stand-in, level {level}, train_frac {train_frac}: sdist at {worst_s:.3f} of its interval's half-width from its middle, tdist {worst_t:.2f} 2^-24")


def reference_sdist(td, wd, anneal, n_new, jitter=None):
    """The reference's own sample_intervals (fp32 torch) on the kernel's exact dilated positions / weights."""
    td_t, wd_t = torch.tensor(td), torch.tensor(wd)
    lg = torch.where(td_t[:, 1:] > td_t[:, :-1], torch.tensor(anneal) * torch.log(wd_t + 0.0), torch.full_like(wd_t, -torch.inf))
    j = None if jitter is None else torch.tensor(jitter)[:, None]
    return mor.sample_intervals(td_t, lg, n_new, j).numpy()


def test_mip_nan_logit_reference_form():
    """train_frac = 0: a non-empty interval with dilated weight 0 gets the logit 0 * log 0 = NaN; the reference's softmax, cumsum and
    sorted_interp then put every centre on the first knot."""
    t = torch.tensor([[0.0, 0.2, 0.5, 0.7, 1.0]])
    w = torch.tensor([[0.3, 0.0, 0.5, 0.2]])
    lg = torch.where(t[:, 1:] > t[:, :-1], 0.0 * torch.log(w + 0.0), torch.full_like(w, -torch.inf))
    assert torch.equal(mor.sample_intervals(t, lg, 8), torch.zeros(1, 9))
    r = sm.mip_resample32(None, None, 0, 8, 0.0, 0.2, 6.0)          # level 0 never sees a NaN: one weight, cdf [0, 1]
    assert not sm.mip_reference_collapse(sm.mip_logits64(r["td"], r["wd"], r["anneal"])).any()


def test_mip_mutants_leave_the_bounds():
    rng = np.random.default_rng(5)
    # `hi > x` as `>=` in the dilation: the interval starting at t1_j = t_j+1 + dilation takes p_j
    worst = 0.0
    for n_prev, n_new in ((8, 16), (33, 31)):
        for kind in ("zero_runs", "onehot"):
            s, w = mip_inputs(128, n_prev, rng, kind)
            bad = sm.mip_resample32(s, w, 1, n_new, 1.0, 0.2, 6.0, mutate="hi_ge")
            td, wd = sm.mip_dilate(s, w, 1)
            c = sm.mip_check(td, wd, bad["anneal"], n_new, bad["sdist"], bad["tdist"], 0.2, 6.0)
            worst = max(worst, float(c["sdist"][~c["collapse"]].max()))
    print(f"\nmip hi >= x: largest sdist fraction of its interval {worst:.3g}")
    assert worst > 1.0
    # kEps dropped from u_max: u moves by up to 2^-23, which only the exact level-0 check sees
    caught = []
    for n_new in (2, 3, 32, 64):
        j = np.array([0.0, 0.5, 1 - 2 ** -24, 0.37], np.float32)
        good = sm.mip_level0_sdist(4, n_new, j)
        bad = sm.mip_resample32(None, np.zeros((4, 1), np.float32), 0, n_new, 0.5, 0.2, 6.0, j, mutate="no_keps")["sdist"]
        ok = sm.mip_resample32(None, np.zeros((4, 1), np.float32), 0, n_new, 0.5, 0.2, 6.0, j)["sdist"]
        assert any(np.array_equal(ok, g) for g in good)
        if not any(np.array_equal(bad, g) for g in good):
            caught.append(n_new)
    print(f"mip kEps dropped from u_max: level-0 sdist off every contraction choice at n_new {caught}")
    assert len(caught) >= 3


# ------------------------------------------------------------------------------------------------ argument checks

@pytest.fixture(scope="module")
def lib():
    from neo360_b200 import build, _lib
    build.build()
    return _lib.load()


def test_sampler_argument_validation_without_gpu(lib):
    """`neo_sample_pdf` rejects NULL t_old / weights / t, an in_sphere other than 0 / 1 and pts / pts_lin without rays_o / rays_d;
    `neo_sample_along_rays` rejects a NULL far (it reads far[b] on every branch) and t -- all before touching the GPU (the pointers
    are never dereferenced)."""
    p = 1 << 20
    pdf = lambda o, d, t_old, w, ins, t, pts, lin: lib.neo_sample_pdf(o, d, None, t_old, w, 4, 9, 8, ins, C.c_float(3.0), None, t, pts,
                                                                      lin, None)
    for args in ((p, p, None, p, 1, p, p, None), (p, p, p, None, 1, p, p, None), (p, p, p, p, 1, None, p, None),
                 (p, p, p, p, 2, p, p, None), (p, p, p, p, -1, p, None, None), (None, p, p, p, 1, p, p, None),
                 (p, None, p, p, 0, p, p, p), (None, None, p, p, 0, p, None, p)):
        assert pdf(*args) == -1, args
    assert b"neo_sample_pdf" in lib.neo_last_error()
    assert lib.neo_sample_pdf(p, p, None, p, p, 4, 3, 8, 1, C.c_float(3.0), None, p, None, None, None) == -1      # n_old < 4
    coarse = lambda o, d, far, ins, t, pts, lin: lib.neo_sample_along_rays(o, d, far, 4, 8, ins, C.c_float(3.0), None, t, pts, lin, None)
    for args in ((p, p, None, 1, p, p, None), (p, p, p, 1, None, p, None), (p, p, p, 2, p, p, None), (None, p, p, 1, p, p, None),
                 (p, None, p, 0, p, p, p)):
        assert coarse(*args) == -1, args
    assert b"neo_sample_along_rays" in lib.neo_last_error()
