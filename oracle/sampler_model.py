"""TEST INFRASTRUCTURE ONLY -- models of the two inverse-CDF resamplers, for holding them to their own arithmetic per sample.

NeO-360 / vanilla NeRF (`resample_kernel`, csrc/sampling.cu):
* `neo_resample(..., rounding=True)` restates the kernel step for step in fp32 numpy: mids, lane-strided partial sums of w[1:-1] and
  the 5-level XOR butterfly, pad / padw / wsum, the pdf by correctly rounded division, the per-32-block Hillis-Steele scan plus the
  carry (lane 31's uncapped value), fminf(1, .), cdf[0] = 0 / cdf[K-1] = 1, prefix max / suffix min of the bins (quirk Q17), the
  kernel's own binary search (its fp32 cdf is not always monotone: two lanes can add the same values in a different association),
  tau with NaN -> 0 and the clamp, the sort, the bg flip, fg pts = o + t d and pts_lin.  Every step is an explicitly rounded IEEE
  operation, so the kernel's t equals this bit for bit.
* `neo_resample(..., rounding=False)` is the same operation in float64 (monotone cdf, searchsorted); it equals
  `neo360_oracle.piecewise_constant_pdf` / `resample_fg` / `resample_bg` / `vanilla_oracle.sample_pdf` in float64.
* `neo_admissible` asks whether each new sample is the float64 operation at some u' with |u' - u| <= eps, give or take delta in
  position.  eps is a priori per ray from the kernel's summation depth: (2 ceil(nw/32) + 16) 2^-24 (the wsum error, one division,
  the 5-level scan and the carry chain); delta = 4 ulp of the bracket's larger end.

Mip-NeRF 360 (`mip::resample_kernel`, csrc/mip.cu): logf / expf are not correctly rounded and nvcc may contract the u formula, the
first / last sdist and s_to_t, so there is no bit-exact emulation.  `mip_dilate` restates the kernel's positions and max-dilated,
renormalised weights exactly (fp32); `mip_check` computes logits, softmax and cdf in float64 with an eps that carries the
exp-of-rounded-logit error, checks every centre's sandwich through the sdist by interval arithmetic and tdist against float64 s_to_t
of the kernel's own sdist.  At level 0 the cdf is exactly [0, 1], so the centres are the kernel's u themselves: `mip_level0_sdist`
gives the kernel's level-0 sdist exactly for each contraction choice of the u formula.
"""
from __future__ import annotations

import math

import numpy as np

F32 = np.float32
U = 2.0 ** -24
KEPS = F32(1.1920929e-07)
DELTA_ULP = 4.0


def f32(x):
    return np.ascontiguousarray(np.asarray(x, dtype=np.float32))


def linspace01(m: int) -> np.ndarray:
    """torch.linspace(0, 1, m) in fp32 as the kernels' `linspace01` computes it (symmetric around the midpoint); it is also
    torch.linspace(0, 1 - 2^-32, m) in fp32, whose end rounds to 1.0 (quirk Q7)."""
    if m == 1:
        return np.zeros(1, F32)
    step = F32(1.0) / F32(m - 1)
    i = np.arange(m)
    lo = step * i.astype(F32)
    hi = F32(1.0) - step * (m - 1 - i).astype(F32)
    return np.where(i < m // 2, lo, hi).astype(F32)


def butterfly_sum(lanes: np.ndarray) -> np.ndarray:
    """warp_sum: (..., 32) lane values -> the value every lane holds after the XOR butterfly (fp32 adds are commutative, so all
    lanes agree)."""
    v = lanes.astype(F32)
    idx = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = v + v[..., idx ^ o]
    return v[..., 0]


def lane_partials(x: np.ndarray) -> np.ndarray:
    """(..., L) -> (..., 32): lane l's `part += x[j]` over j = l, l + 32, ... in order, starting from 0."""
    L = x.shape[-1]
    part = np.zeros(x.shape[:-1] + (32,), F32)
    for base in range(0, L, 32):
        blk = x[..., base:base + 32]
        part[..., :blk.shape[-1]] = part[..., :blk.shape[-1]] + blk
    return part


def block_scan(v: np.ndarray, drop_carry_at: int = -1) -> np.ndarray:
    """Inclusive per-32-block Hillis-Steele scan plus carry, as `warp_incl_scan_add` + `add_(., carry)`; returns the uncapped sums.
    `drop_carry_at` (mutation only) restarts the carry at that block."""
    n = v.shape[-1]
    out = np.empty_like(v, dtype=F32)
    carry = np.zeros(v.shape[:-1], F32)
    for bi, base in enumerate(range(0, n, 32)):
        blk = np.zeros(v.shape[:-1] + (32,), F32)
        w = min(32, n - base)
        blk[..., :w] = v[..., base:base + w]
        for o in (1, 2, 4, 8, 16):
            sh = blk.copy()
            sh[..., o:] = blk[..., :-o]
            blk = np.where(np.arange(32) >= o, blk + sh, blk).astype(F32)
        if bi == drop_carry_at:
            carry = np.zeros_like(carry)
        sc = blk + carry[..., None]
        out[..., base:base + w] = sc[..., :w]
        carry = sc[..., 31]
    return out


def search(cdf: np.ndarray, u: np.ndarray, strict: bool = False) -> np.ndarray:
    """The kernels' binary search, probe for probe: lo = 0, hi = K; while hi - lo > 1: mid; cdf[mid] <= u ? lo = mid : hi = mid."""
    K = cdf.shape[-1]
    lo = np.zeros(u.shape, np.int64)
    hi = np.full(u.shape, K, np.int64)
    rows = np.arange(u.shape[0])[:, None]
    while True:
        act = hi - lo > 1
        if not act.any():
            return lo
        mid = (lo + hi) >> 1
        c = cdf[rows, np.minimum(mid, K - 1)]
        ok = (c < u) if strict else (c <= u)
        lo = np.where(act & ok, mid, lo)
        hi = np.where(act & ~ok, mid, hi)


# ------------------------------------------------------------------------------------------------ NeO-360 / vanilla NeRF

def neo_cdf32(t_old, w, mutate=None):
    """Kernel bins (K) and fp32 cdf (K) of each ray.  `mutate` names a planted bug (tests of the tests only)."""
    t_old, w = f32(t_old), f32(w)
    K = t_old.shape[-1] - 1
    nw = K - 1
    bins = (F32(0.5) * (t_old[:, 1:] + t_old[:, :-1])).astype(F32)
    ww = w[:, 0:nw] if mutate == "w_shift" else w[:, 1:1 + nw]
    wsum = butterfly_sum(lane_partials(ww))
    pad = np.maximum(F32(0.0), F32(1e-5) - wsum).astype(F32)
    padw = (pad / F32(nw + 1 if mutate == "pad_count" else nw)).astype(F32)
    wsum = (wsum + pad).astype(F32)
    with np.errstate(divide="ignore", invalid="ignore"):
        pdf = ((ww[:, :nw - 1] + padw[:, None]) / wsum[:, None]).astype(F32)
    sc = block_scan(pdf, drop_carry_at=1 if mutate == "carry" else -1)
    cdf = np.empty((t_old.shape[0], K), F32)
    cdf[:, 1:K - 1] = np.fmin(F32(1.0), sc)
    cdf[:, 0], cdf[:, K - 1] = 0.0, 1.0
    return bins, cdf


def neo_u(n, m, u_rand=None, mutate=None):
    if u_rand is not None:
        return f32(u_rand)
    if mutate == "no_q7":        # linspace(0, 1 - 2^-32, m) without the endpoint rounding to 1.0f
        u = np.linspace(0.0, 1.0 - 2.0 ** -32, m).astype(F32)
        u[-1] = np.nextafter(F32(1.0), F32(0.0))
    else:
        u = linspace01(m)
    return np.broadcast_to(u, (n, m)).copy()


def neo_new_samples32(t_old, w, m, u_rand=None, mutate=None):
    """The kernel's new samples in u order (before the sort), its u, bins and cdf."""
    bins, cdf = neo_cdf32(t_old, w, mutate)
    n, K = bins.shape
    u = neo_u(n, m, u_rand, mutate)
    pmax = np.maximum.accumulate(bins, axis=-1)
    smin = np.minimum.accumulate(bins[:, ::-1], axis=-1)[:, ::-1]
    lo = search(cdf, u, strict=(mutate == "strict_search"))
    rows = np.arange(n)[:, None]
    last = lo + 1 >= K
    up = np.minimum(lo + 1, K - 1)
    c0 = cdf[rows, lo]
    c1 = np.where(last, cdf[:, K - 1:K], cdf[rows, up])
    if mutate == "q17_neighbours":
        b0 = bins[rows, lo]
        b1 = np.where(last, bins[:, K - 1:K], bins[rows, up])
    else:
        b0 = pmax[rows, lo]
        b1 = np.where(last, bins[:, K - 1:K], smin[rows, up])
    with np.errstate(divide="ignore", invalid="ignore"):
        tau = ((u - c0) / (c1 - c0)).astype(F32)
    tau = np.where(np.isnan(tau), F32(0.0), tau)
    tau = np.minimum(np.maximum(tau, F32(0.0)), F32(1.0)).astype(F32)
    x = (b0 + tau * (b1 - b0)).astype(F32)
    return x, u, bins, cdf


def ray_far32(o, d):
    """ray_geom's g.far (intersect_sphere) in the kernel's fp32 operation order."""
    o, d = f32(o), f32(d)
    dot = lambda a, b: ((a[:, 0] * b[:, 0] + a[:, 1] * b[:, 1]).astype(F32) + a[:, 2] * b[:, 2]).astype(F32)
    dd = dot(d, d)
    d1 = (-dot(d, o) / dd).astype(F32)
    p = (o + d1[:, None] * d).astype(F32)
    inv = (F32(1.0) / np.sqrt(dd)).astype(F32)
    p2 = dot(p, p)
    return (d1 + np.sqrt(F32(1.0) - p2) * inv).astype(F32)


def neo_resample(t_old, w, m, in_sphere, u_rand=None, o=None, d=None, far_unc=3.0, rounding=True, mutate=None):
    """`neo_sample_pdf`: returns dict(t (n, n_old+m) sorted -- descending for bg --, new (n, m) in u order, u, pts / pts_lin when
    o, d are given).  rounding=False is the float64 operation (no pts)."""
    if not rounding:
        t_old, w = np.asarray(t_old, np.float64), np.asarray(w, np.float64)
        bins = 0.5 * (t_old[:, 1:] + t_old[:, :-1])
        n = t_old.shape[0]
        # the reference draws its deterministic u as an fp32 linspace even for float64 weights (helper.py:194)
        u = np.asarray(u_rand if u_rand is not None else np.broadcast_to(linspace01(m), (n, m)), np.float64)
        x = pdf_samples64(bins, w[:, 1:-1], u)
        t = np.sort(np.concatenate([t_old, x], -1), -1)
        return dict(t=t if in_sphere else t[:, ::-1], new=x, u=u)
    x, u, bins, cdf = neo_new_samples32(t_old, w, m, u_rand, mutate)
    t = np.sort(np.concatenate([f32(t_old), x], -1), -1)
    if not in_sphere:
        t = t[:, ::-1]
    out = dict(t=np.ascontiguousarray(t), new=x, u=u, bins=bins, cdf=cdf)
    if o is not None:
        o32, d32 = f32(o), f32(d)
        if in_sphere:
            out["pts"] = (o32[:, None, :] + t[..., None] * d32[:, None, :]).astype(F32)
        else:
            far = ray_far32(o32, d32)
            tl = (far[:, None] * (F32(1.0) - t) + F32(far_unc) * t).astype(F32)
            out["pts_lin"] = (o32[:, None, :] + tl[..., None] * d32[:, None, :]).astype(F32)
    return out


def cdf64(w):
    """[0, min(1, cumsum(pdf[:-1])), 1] of the padded weights in float64 (helper.py:174-215)."""
    import torch           # its float64 sum / cumsum order, so that the float64 form is the oracle's to the last bits
    w = torch.from_numpy(np.asarray(w, np.float64))
    wsum = w.sum(-1, keepdim=True)
    pad = torch.fmax(torch.zeros_like(wsum), 1e-5 - wsum)
    pdf = (w + pad / w.shape[-1]) / (wsum + pad)
    c = np.fmin(1.0, torch.cumsum(pdf[:, :-1], -1).numpy())
    return np.concatenate([np.zeros_like(c[:, :1]), c, np.ones_like(c[:, :1])], -1)


def pdf_samples64(bins, w, u):
    """piecewise_constant_pdf in float64 with its value max / min bracket (Q17): lo = last j with cdf[j] <= u."""
    bins, u = np.asarray(bins, np.float64), np.asarray(u, np.float64)
    cdf = cdf64(w)
    n, K = bins.shape
    rows = np.arange(n)[:, None]
    lo = np.clip(rsearch(cdf, u, "right") - 1, 0, K - 1)
    last = lo + 1 >= K
    up = np.minimum(lo + 1, K - 1)
    pmax = np.maximum.accumulate(bins, axis=-1)
    smin = np.minimum.accumulate(bins[:, ::-1], axis=-1)[:, ::-1]
    c0, c1 = cdf[rows, lo], np.where(last, 1.0, cdf[rows, up])
    b0, b1 = pmax[rows, lo], np.where(last, bins[:, K - 1:K], smin[rows, up])
    with np.errstate(divide="ignore", invalid="ignore"):
        tau = (u - c0) / (c1 - c0)
    tau = np.clip(np.nan_to_num(tau, nan=0.0), 0.0, 1.0)
    return b0 + tau * (b1 - b0)


def neo_eps(n_old: int) -> float:
    nw = n_old - 2
    return (2 * math.ceil(nw / 32) + 16) * U


def rsearch(a, v, side="right"):
    """Row-wise searchsorted of v (n, m) in the non-decreasing rows of a (n, K): the number of a[j] <= v (right) or < v (left)."""
    K = a.shape[1]
    lo = np.zeros(v.shape, np.int64)
    hi = np.full(v.shape, K, np.int64)
    rows = np.arange(a.shape[0])[:, None]
    while (lo < hi).any():
        mid = (lo + hi) >> 1
        x = a[rows, np.minimum(mid, K - 1)]
        act = lo < hi
        go = (x <= v) if side == "right" else (x < v)
        lo, hi = np.where(act & go, mid + 1, lo), np.where(act & ~go, mid, hi)
    return lo


def inv_lo(x, cdf, v):
    """inf { y : G(y) >= v } of the piecewise-linear G through (x_j, cdf_j), x ascending, cdf non-decreasing (per ray)."""
    j = rsearch(cdf, v, "left")
    rows = np.arange(x.shape[0])[:, None]
    jj = np.clip(j, 1, x.shape[1] - 1)
    c0, c1, x0, x1 = cdf[rows, jj - 1], cdf[rows, jj], x[rows, jj - 1], x[rows, jj]
    with np.errstate(divide="ignore", invalid="ignore"):
        y = x0 + np.clip(np.nan_to_num((v - c0) / (c1 - c0), nan=1.0), 0, 1) * (x1 - x0)
    return np.where(j <= 0, x[:, :1], np.where(j >= x.shape[1], x[:, -1:], y))


def inv_hi(x, cdf, v):
    """sup { y : G(y) <= v }."""
    j = rsearch(cdf, v, "right") - 1
    rows = np.arange(x.shape[0])[:, None]
    jj = np.clip(j, 0, x.shape[1] - 2)
    c0, c1, x0, x1 = cdf[rows, jj], cdf[rows, jj + 1], x[rows, jj], x[rows, jj + 1]
    with np.errstate(divide="ignore", invalid="ignore"):
        y = x0 + np.clip(np.nan_to_num((v - c0) / (c1 - c0), nan=0.0), 0, 1) * (x1 - x0)
    return np.where(j < 0, x[:, :1], np.where(j >= x.shape[1] - 1, x[:, -1:], y))


def sandwich(x, cdf, u, eps):
    """[G^-1(u - eps) - delta, G^-1(u + eps) + delta] with flat runs' preimages taken whole; delta = 4 ulp of the larger end."""
    lo = inv_lo(x, cdf, u - eps)
    hi = inv_hi(x, cdf, u + eps)
    delta = DELTA_ULP * U * np.maximum(np.abs(lo), np.abs(hi))
    return lo - delta, hi + delta


def G(x, cdf, y):
    """The float64 cdf as a function of position: right-continuous piecewise-linear through (x_j, cdf_j), x ascending."""
    j = rsearch(x, y, "right") - 1
    rows = np.arange(x.shape[0])[:, None]
    jj = np.clip(j, 0, x.shape[1] - 2)
    x0, x1, c0, c1 = x[rows, jj], x[rows, jj + 1], cdf[rows, jj], cdf[rows, jj + 1]
    with np.errstate(divide="ignore", invalid="ignore"):
        g = c0 + np.clip((y - x0) / (x1 - x0), 0, 1) * (c1 - c0)
    return np.where(j < 0, 0.0, np.where(j >= x.shape[1] - 1, 1.0, g))


def neo_admissible(t_old, w, new, u, in_sphere):
    """Per new sample, the fraction of eps it needs (<= 1 is admissible) to be the float64 operation at some u' with |u' - u| <= eps,
    give or take delta = 4 ulp of the bracket's larger end in position.

    fg / vanilla (ascending bins, monotone G): the sandwich x in [G^-1(u - eps) - delta, G^-1(u + eps) + delta], i.e.
    G(x + delta) >= u - eps and G(x - delta) <= u + eps; flat runs of G have their whole preimage, so no case split for bracket flips.
    bg (descending bins, Q17: every sample is bins[0] + tau (bins[K-1] - bins[0])): tau (widened by delta) is mapped back to
    u' = c0 + tau (c1 - c0) in each bracket within u +- eps; the value is the least |u' - u| / eps."""
    t_old, w = np.asarray(t_old, np.float64), np.asarray(w, np.float64)
    new, u = np.asarray(new, np.float64), np.asarray(u, np.float64)
    bins = 0.5 * (t_old[:, 1:] + t_old[:, :-1])
    cdf = cdf64(w[:, 1:-1])
    eps = neo_eps(t_old.shape[1])
    rows = np.arange(bins.shape[0])[:, None]
    K = bins.shape[1]
    if in_sphere:
        j = np.clip(rsearch(bins, new, "right") - 1, 0, K - 2)
        delta = DELTA_ULP * U * np.maximum(np.abs(bins[rows, j]), np.abs(bins[rows, j + 1]))
        need = np.maximum(0.0, np.maximum(u - G(bins, cdf, new + delta), G(bins, cdf, new - delta) - u))
        return need / eps
    b0, bK = bins[:, :1], bins[:, -1:]
    span = bK - b0
    delta = DELTA_ULP * U * np.maximum(np.abs(b0), np.abs(bK))
    with np.errstate(divide="ignore", invalid="ignore"):
        ta = np.where(span != 0, (new - delta - b0) / span, 0.0)
        tb = np.where(span != 0, (new + delta - b0) / span, 1.0)
    tlo, thi = np.clip(np.minimum(ta, tb), 0, 1), np.clip(np.maximum(ta, tb), 0, 1)
    # brackets [c_j, c_j+1] that meet [u - eps, u + eps]; with eps' = 64 eps the catalogue's mutants still get a finite distance
    wide = 64 * eps
    jl = np.clip(rsearch(cdf, u - wide, "left") - 1, 0, K - 2)
    jh = np.clip(rsearch(cdf, u + wide, "right") - 1, 0, K - 2)
    best = np.full(new.shape, np.inf)
    for off in range(int((jh - jl).max()) + 1):
        jj = np.minimum(jl + off, jh)
        c0, c1 = cdf[rows, jj], cdf[rows, jj + 1]
        ulo, uhi = c0 + tlo * (c1 - c0), c0 + thi * (c1 - c0)
        best = np.minimum(best, np.maximum(0.0, np.maximum(ulo - u, u - uhi)))
    # u = 1 takes the degenerate last bracket (c0 = c1 = 1, tau = 0/0 -> 0): the sample is bins[0]
    best = np.where(tlo <= 0.0, np.minimum(best, np.abs(1.0 - u)), best)
    return best / eps


FAMILIES = ["rand4", "uniform", "onehot_first", "onehot_last", "onehot_mid", "ends_only", "zero", "sum_below", "sum_at",
            "sum_above", "zero_runs", "rand16", "unnormalised", "dup_t"]


def weight_family(fam, n, n_old, rng):
    """(t ascending in [0.01, 6], w) of one weight family; ends_only puts mass only in the excluded w[0] / w[-1]."""
    t = np.sort(0.01 + 6 * rng.random((n, n_old)), -1).astype(np.float32)
    w = np.zeros((n, n_old), np.float32)
    K = n_old - 1
    if fam == "rand4":
        w = (rng.random((n, n_old)) ** 4).astype(np.float32)
    elif fam == "uniform":
        w[:] = 1.0 / n_old
    elif fam.startswith("onehot"):
        j = {"onehot_first": 1, "onehot_last": n_old - 2, "onehot_mid": n_old // 2}[fam]
        w[:, j] = 1.0
    elif fam == "ends_only":
        w[:, 0], w[:, -1] = 0.7, 0.3
    elif fam.startswith("sum_"):
        s = {"sum_below": np.float32(0.99e-5), "sum_at": np.float32(1e-5), "sum_above": np.float32(1.01e-5)}[fam]
        w[:, 1:-1] = rng.random((n, n_old - 2))
        w[:, 1:-1] = (w[:, 1:-1] / w[:, 1:-1].sum(-1, keepdims=True) * s).astype(np.float32)
    elif fam == "zero_runs":
        w = (rng.random((n, n_old)) ** 4).astype(np.float32)
        L = max(1, K // 5)
        w[:, 1:1 + L] = 0.0
        w[:, K // 2 - L // 2:K // 2 + L // 2 + 1] = 0.0
        w[:, -1 - L:] = 0.0
        w[rng.random((n, n_old)) < 0.3] = 0.0
    elif fam == "rand16":
        w = (rng.random((n, n_old)) ** 16).astype(np.float32)
    elif fam == "unnormalised":
        w = (rng.random((n, n_old)) * 1e3 / n_old * rng.random((n, 1)) * 2).astype(np.float32)
    elif fam == "dup_t":
        w = (rng.random((n, n_old)) ** 4).astype(np.float32)
        j = np.arange(1, n_old, 3)
        t[:, j] = t[:, j - 1]
    return t, w



# ------------------------------------------------------------------------------------------------ Mip-NeRF 360

def mip_dilation(level: int, n_prev: int) -> np.float32:
    prod = F32(1.0)
    for _ in range(level):
        prod = F32(prod * F32(n_prev))
    return F32(F32(0.0025) + F32(0.5) / prod)


def mip_anneal(train_frac: float) -> np.float32:
    tf = F32(train_frac)
    return F32(F32(F32(10.0) * tf) / F32(F32(F32(9.0) * tf) + F32(1.0)))


def mip_dilate(s_prev, w_prev, level, mutate=None):
    """The kernel's positions td (n, ns) and renormalised dilated weights wd (n, ns - 1), both fp32 and exact: dilation, sort, clip,
    max over the covering intervals (t0_j <= x < t1_j), p * dt, lane-strided + butterfly total, drop first / last."""
    if level == 0:
        n = w_prev.shape[0] if w_prev is not None else (s_prev.shape[0] if s_prev is not None else 1)
        return np.broadcast_to(np.array([0.0, 1.0], F32), (n, 2)).copy(), np.ones((n, 1), F32)
    t, w = f32(s_prev), f32(w_prev)
    n, npv = w.shape
    dil = mip_dilation(level, npv)
    a, c = t[:, :-1], t[:, 1:]
    pp = (w / np.maximum((c - a).astype(F32), KEPS)).astype(F32)
    lo, hi = (a - dil).astype(F32), (c + dil).astype(F32)
    td = np.sort(np.concatenate([t, lo, hi], -1), -1)
    td = np.minimum(np.maximum(td, F32(0.0)), F32(1.0)).astype(F32)
    total = td.shape[1]
    x = td[:, :-1]
    cov = (lo[:, None, :] <= x[:, :, None]) & ((hi[:, None, :] >= x[:, :, None]) if mutate == "hi_ge" else (hi[:, None, :] > x[:, :, None]))
    m = np.where(cov, pp[:, None, :], F32(0.0)).max(-1).astype(F32)
    wv = (m * (td[:, 1:] - x).astype(F32)).astype(F32)
    tot = np.maximum(butterfly_sum(lane_partials(wv)), KEPS).astype(F32)
    wd = (wv[:, 1:total - 2] / tot[:, None]).astype(F32)
    return np.ascontiguousarray(td[:, 1:total - 1]), np.ascontiguousarray(wd)


def mip_u64(n_rays, n_new, jitter=None):
    """sample_intervals' u (helper.py:343-396) in float64; jitter (n_rays,) fp32 or None."""
    eps = float(KEPS)
    if jitter is None:
        pad = 1 / (2 * n_new)
        return np.broadcast_to(np.linspace(pad, 1 - pad - eps, n_new), (n_rays, n_new)).copy()
    u_max = eps + (1 - eps) / n_new
    mj = (1 - u_max) / (n_new - 1) - eps
    return np.linspace(0, 1 - u_max, n_new)[None, :] + np.asarray(jitter, np.float64)[:, None] * mj


def _fma32(a, b, c):
    return (np.asarray(a, np.longdouble) * np.asarray(b, np.longdouble) + np.asarray(c, np.longdouble)).astype(F32)


def mip_u32(n_rays, n_new, jitter=None, fuse_base=False, fuse_u=False, mutate=None):
    """The kernel's fp32 u for one choice of contraction of `end - step * m` / `start + step * k` and `base + jitter * max_jitter`."""
    k = np.arange(n_new)
    kf, mf = k.astype(F32), (n_new - 1 - k).astype(F32)
    half = k < n_new // 2
    nn = F32(n_new)
    if jitter is not None:
        u_max = (F32(1.0) / nn) if mutate == "no_keps" else F32(KEPS + F32(F32(F32(1.0) - KEPS) / nn))
        mj = F32(F32(F32(F32(1.0) - u_max) / F32(n_new - 1)) - KEPS)
        end = F32(F32(1.0) - u_max)
        step = F32(end / F32(n_new - 1))
        hi = _fma32(-step, mf, end) if fuse_base else (end - (step * mf).astype(F32)).astype(F32)
        base = np.where(half, (step * kf).astype(F32), hi)
        j = f32(jitter)[:, None]
        return _fma32(j, mj, base[None]) if fuse_u else (base[None] + (j * mj).astype(F32)).astype(F32)
    pad = F32(F32(1.0) / F32(F32(2.0) * nn))
    start, end = pad, F32(F32(F32(1.0) - pad) - KEPS)
    step = F32(F32(end - start) / F32(n_new - 1))
    if fuse_base:
        lo_, hi_ = _fma32(step, kf, start), _fma32(-step, mf, end)
    else:
        lo_, hi_ = (start + (step * kf).astype(F32)).astype(F32), (end - (step * mf).astype(F32)).astype(F32)
    return np.broadcast_to(np.where(half, lo_, hi_).astype(F32), (n_rays, n_new)).copy()


def mip_sdist_from_centres32(c):
    """The kernel's sdist from fp32 centres (2 c0 is exact, so fused or not the first / last are the same)."""
    c = f32(c)
    mid = (F32(0.5) * (c[:, 1:] + c[:, :-1]).astype(F32)).astype(F32)
    first = np.maximum((F32(2.0) * c[:, :1] - mid[:, :1]).astype(F32), F32(0.0))
    last = np.minimum((F32(2.0) * c[:, -1:] - mid[:, -1:]).astype(F32), F32(1.0))
    return np.concatenate([first, mid, last], -1).astype(F32)


def mip_level0_sdist(n_rays, n_new, jitter=None, mutate=None):
    """Level 0: cdf = [0, 1] and td = [0, 1] exactly, so every centre is the kernel's u.  Returns the sdist of every contraction
    choice (a list)."""
    return [mip_sdist_from_centres32(mip_u32(n_rays, n_new, jitter, fb, fu, mutate)) for fb in (False, True) for fu in (False, True)]


def mip_logits64(td, wd, anneal):
    nonempty = td[:, 1:] > td[:, :-1]
    with np.errstate(divide="ignore", invalid="ignore"):
        lg = np.where(nonempty, float(anneal) * np.log(np.asarray(wd, np.float64)), -np.inf)
    return lg


def mip_reference_collapse(lg):
    """Rays on which the reference's softmax is NaN and its sorted_interp puts every centre on the first knot: a NaN logit
    (0 * log 0 at anneal 0) or every logit -inf, with at least two weights (with one weight the cdf is [0, 1] whatever the softmax)."""
    return (np.isnan(lg).any(-1) | np.isneginf(lg).all(-1)) & (lg.shape[1] >= 2)


def mip_cdf64_eps(td, wd, anneal):
    """float64 softmax cdf (ns) and the a-priori eps per ray.  eps carries, per weight, the exp of the kernel's rounded logit:
    the logit anneal * logf(w) has relative error <= 2 2^-24, the difference to the max adds |l_j| + |l_max| of it and 2^-24 |l_j - l_max|
    for its own rounding, expf adds 2 ulp and the division 1; the total se and the scan add (2 ceil(nw/32) + 12) 2^-24, and u's own
    rounding against the float64 linspace / jitter formula 8 2^-24."""
    lg = mip_logits64(td, wd, anneal)
    n, nw = lg.shape
    fin = np.isfinite(lg)
    mx = np.where(fin, lg, -np.inf).max(-1, keepdims=True)
    mxs = np.where(np.isfinite(mx), mx, 0.0)
    with np.errstate(invalid="ignore"):
        e = np.where(fin, np.exp(np.where(fin, lg, 0.0) - mxs), 0.0)
    se = e.sum(-1, keepdims=True)
    p = e / np.where(se > 0, se, 1.0)
    spread = np.where(fin, 2 * (np.abs(lg) + np.abs(mxs)) + np.abs(lg - mxs) + 3, 0.0)
    eps = (2 * (p * np.where(fin, spread, 0.0)).sum(-1) + 2 * math.ceil(nw / 32) + 12 + 8) * U
    c = np.fmin(1.0, np.cumsum(p[:, :-1], -1))
    cdf = np.concatenate([np.zeros((n, 1)), c, np.ones((n, 1))], -1)
    return cdf, eps, lg


def mip_check(td, wd, anneal, n_new, sdist, tdist, near, far, jitter=None):
    """Fraction of each bound the kernel's sdist / tdist use (<= 1 passes), over the rays whose reference softmax is finite:
    returns dict(sdist=(n, n_new+1) fraction, tdist=(n, n_new+1) relative error / 2^-24, collapse=(n,) bool)."""
    td64 = np.asarray(td, np.float64)
    cdf, eps, lg = mip_cdf64_eps(td, wd, anneal)
    u = mip_u64(td.shape[0], n_new, jitter)
    e = eps[:, None]
    clo, chi = sandwich(td64, cdf, u, e)
    s = np.asarray(sdist, np.float64)
    rnd = 4 * U
    lo = np.concatenate([np.maximum(1.5 * clo[:, :1] - 0.5 * chi[:, 1:2], 0.0), 0.5 * (clo[:, 1:] + clo[:, :-1]),
                         np.minimum(1.5 * clo[:, -1:] - 0.5 * chi[:, -2:-1], 1.0)], -1)
    hi = np.concatenate([np.maximum(1.5 * chi[:, :1] - 0.5 * clo[:, 1:2], 0.0), 0.5 * (chi[:, 1:] + chi[:, :-1]),
                         np.minimum(1.5 * chi[:, -1:] - 0.5 * clo[:, -2:-1], 1.0)], -1)
    lo, hi = lo - rnd * np.abs(lo) - rnd, hi + rnd * np.abs(hi) + rnd
    # how far outside [lo, hi] each sdist lies, in units of the interval's half-width beyond its centre (> 1 fails)
    mid, half = 0.5 * (lo + hi), 0.5 * (hi - lo)
    frac = np.abs(s - mid) / np.maximum(half, 1e-300)
    t_ref = 1.0 / (s * (1.0 / far) + (1.0 - s) * (1.0 / near))
    trel = np.abs(np.asarray(tdist, np.float64) - t_ref) / np.abs(t_ref) / U
    return dict(sdist=frac, tdist=trel, collapse=mip_reference_collapse(lg))


def mip_resample32(s_prev, w_prev, level, n_new, train_frac, near, far, jitter=None, mutate=None):
    """An fp32 numpy stand-in for the whole kernel (np.log / np.exp for logf / expf, no contraction), for the CPU checks of the bounds
    and of the mutation catalogue.  It follows the reference form on NaN / all -inf logits (every centre on the first knot)."""
    td, wd = mip_dilate(s_prev, w_prev, level, mutate)
    n, ns = td.shape
    nw = ns - 1
    an = mip_anneal(train_frac)
    with np.errstate(divide="ignore", invalid="ignore"):
        lg = np.where(td[:, 1:] > td[:, :-1], (an * np.log(wd)).astype(F32), F32(-np.inf)).astype(F32)
        mx = np.fmax.reduce(lg, axis=-1, keepdims=True)
        e = np.exp((lg - mx).astype(F32)).astype(F32)
    se = butterfly_sum(lane_partials(e))
    cw = np.empty((n, ns), F32)
    if nw >= 2:
        with np.errstate(divide="ignore", invalid="ignore"):
            pdf = (e[:, :nw - 1] / se[:, None]).astype(F32)
        cw[:, 1:ns - 1] = np.fmin(block_scan(pdf), F32(1.0))
    cw[:, 0], cw[:, ns - 1] = 0.0, 1.0
    u = mip_u32(n, n_new, jitter, mutate=mutate)
    a = search(cw, u)
    rows = np.arange(n)[:, None]
    last = a + 1 >= ns
    up = np.minimum(a + 1, ns - 1)
    x0, x1 = cw[rows, a], np.where(last, cw[:, ns - 1:], cw[rows, up])
    f0, f1 = td[rows, a], np.where(last, td[:, ns - 1:], td[rows, up])
    with np.errstate(divide="ignore", invalid="ignore"):
        off = ((u - x0) / (x1 - x0)).astype(F32)
    off = np.minimum(np.maximum(np.where(np.isnan(off), F32(0.0), off), F32(0.0)), F32(1.0))
    c = (f0 + off * (f1 - f0)).astype(F32)
    collapse = (np.isnan(se)) & (nw >= 2)
    c = np.where(collapse[:, None], td[:, :1], c)
    s = mip_sdist_from_centres32(c)
    sn, sf = F32(1.0) / F32(near), F32(1.0) / F32(far)
    t = (F32(1.0) / (s * sf + (F32(1.0) - s) * sn).astype(F32)).astype(F32)
    return dict(sdist=s, tdist=t, td=td, wd=wd, anneal=an)
