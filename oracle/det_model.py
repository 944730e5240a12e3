"""Models of the deterministic training kernels (csrc/det.cu) and their a-priori error bounds.

* segment_emulate: the order-fixed scatter of `neo_index_maps_bwd_det` / `neo_grid_encoder_features_bwd_det` restated step for step in
  fp32 over the kernel's own sorted entries: per texel, acc = acc + w * g (each product and sum rounded to fp32) in sorted order, starting
  from the map's value.  The kernel must match it bit for bit.  scatter_bound: |fp32 sum - exact| <= (n + 1) 2^-24 (sum |w g| + |start|)
  for a texel of n entries (sequential summation; every product's own rounding included).
* distortion64 / distortion_grad64: `training.distortion_loss` per ray and its gradient in float64, the formula as written (for descending m
  the pair term is minus sum w_i w_j |m_i - m_j|).  distortion_bounds: a-priori bounds of the kernels' fp32 results.
* interlevel64 / interlevel_grad64: one proposal level of `mip.training_loss`'s interlevel term per ray and its gradient with respect to the
  proposal weights, with `mip._outer_weights`' searchsorted(right=True) / lo / hi semantics.  interlevel_bounds: a-priori bounds.
* upsample_matrix / upsample64 / upsample_adjoint64: F.interpolate(bilinear, align_corners=True) as a matrix per axis, with ATen's tap
  weights computed in fp32 (as the kernel does) or float64 (as autograd in float64 does); upsample_bound: a-priori bound of the kernel.
"""
from __future__ import annotations

import numpy as np
import torch

U = 2.0 ** -24


# ---- order-fixed scatter ----

def workspace_offsets(E: int, T: int):
    """Byte offsets of the workspace blocks (include/neo360_b200.h): keys, keys_sorted, ids, ids_sorted, wts, starts."""
    off, out = 0, {}
    for name, n in (("keys", E), ("keys_sorted", E), ("ids", E), ("ids_sorted", E), ("wts", E), ("starts", T + 1)):
        out[name] = off
        off += (4 * n + 255) // 256 * 256
    return out


def read_entries(ws: torch.Tensor, E: int, T: int):
    """(sorted keys, sorted entry ids, weights by entry id) of a workspace after a call, as int64 / float32 tensors."""
    o = workspace_offsets(E, T)
    view = lambda name, n, dt: ws[o[name]:o[name] + 4 * n].view(dt)
    ks = view("keys_sorted", E, torch.int32).long() & 0xFFFFFFFF
    ids = view("ids_sorted", E, torch.int32).long() & 0xFFFFFFFF
    return ks, ids, view("wts", E, torch.float32).clone()


def segment_emulate(keys, ids, wts, g_of, init, reverse=False):
    """fp32 restatement of segment_reduce_kernel.  keys / ids (E,) sorted; wts (E,) by entry id; g_of(entry ids) -> (k, C) fp32 = their
    row gradients; init (T, C) fp32 = the maps' values before the call.  Returns (T, C) fp32.  Entries with key >= T are not summed.
    `reverse` sums each segment in reverse order (a mutant)."""
    T = init.shape[0]
    keep = keys < T
    keys, ids = keys[keep], ids[keep]
    out = init.clone()
    if keys.numel() == 0:
        return out
    uniq, counts = torch.unique_consecutive(keys, return_counts=True)
    starts = torch.cumsum(counts, 0) - counts
    acc = out[uniq].clone()
    for j in range(int(counts.max())):
        act = counts > j
        pos = torch.where(act, starts + (counts - 1 - j if reverse else j), torch.zeros_like(starts))[act]
        e = ids[pos]
        acc[act] = acc[act] + wts[e][:, None] * g_of(e)          # fp32: product rounded, then the sum rounded
    out[uniq] = acc
    return out


def scatter_exact(keys, ids, wts, g_of, init):
    """float64 value of the same sums and the bound's magnitude: (val, mag, n) per texel."""
    T, C = init.shape
    keep = keys < T
    keys, ids = keys[keep], ids[keep]
    val = init.double().clone()
    mag = init.double().abs().clone()
    n = torch.zeros(T, dtype=torch.float64, device=init.device)
    wg = wts[ids].double()[:, None] * g_of(ids).double()
    val.index_add_(0, keys, wg)
    mag.index_add_(0, keys, wg.abs())
    n.index_add_(0, keys, torch.ones_like(keys, dtype=torch.float64))
    return val, mag, n


def scatter_bound(mag, n):
    return (n[:, None] + 1) * U * mag


# ---- distortion loss ----

def distortion64(w, m, I):
    """Per-ray 1/3 sum I w^2 + 2 sum_k (w_k m_k W_<k - w_k (wm)_<k), float64."""
    w, m, I = (t.double() for t in (w, m, I))
    wm = w * m
    W_lt = torch.cumsum(w, -1) - w
    WM_lt = torch.cumsum(wm, -1) - wm
    return (I * w * w).sum(-1) / 3 + 2 * (wm * W_lt - w * WM_lt).sum(-1)


def distortion_grad64(w, m, I, g):
    """d distortion64 / d w times the per-ray upstream g, float64."""
    w, m, I, g = (t.double() for t in (w, m, I, g))
    wm = w * m
    W_lt, WM_lt = torch.cumsum(w, -1) - w, torch.cumsum(wm, -1) - wm
    W_gt, WM_gt = w.sum(-1, keepdim=True) - W_lt - w, wm.sum(-1, keepdim=True) - WM_lt - wm
    return (2.0 / 3.0 * I * w + 2 * (m * W_lt - WM_lt + WM_gt - m * W_gt)) * g[..., None]


def distortion_bounds(w, m, I, g):
    """A-priori bounds of the kernels' fp32 results: loss (n,), grad (n,N).  The kernel's sums are chunked scans of depth <= N/32 + 5 plus a
    five-level butterfly, so every computed partial sum carries at most (N + 64) 2^-24 relative to its absolute terms."""
    w, m, I, g = (t.double().abs() for t in (w, m, I, g))
    N = w.shape[-1]
    k = (N + 64) * U
    tw, twm = w.sum(-1, keepdim=True), (w * m).sum(-1, keepdim=True)
    loss = k * 4 * ((I * w * w).sum(-1) / 3 + 2 * (2 * w * m * tw + 2 * w * twm).sum(-1))
    grad = k * 4 * (2.0 / 3.0 * I * w + 2 * (4 * m * tw + 4 * twm)) * g[..., None]
    return loss, grad


# ---- interlevel loss ----
EPS = 1.1920929e-07


def outer_ranges(c, t_env):
    """lo_j, hi_{j+1} of mip._outer_weights for every interval j of c (n, Nc+1) against t_env (n, Np+1)."""
    r = torch.searchsorted(t_env.contiguous(), c.contiguous(), right=True)
    lo, hi = (r - 1).clamp(min=0), r.clamp(max=t_env.shape[-1] - 1)
    return lo[..., :-1], hi[..., 1:]


def outer64(c, t_env, w_env, short=False):
    """w_outer_j = sum of w_env over [lo_j, hi_{j+1}) in float64 ([lo_j, hi_j) with `short`, a mutant)."""
    lo, hi = outer_ranges(c, t_env)
    if short:
        r = torch.searchsorted(t_env.contiguous(), c.contiguous(), right=True).clamp(max=t_env.shape[-1] - 1)
        hi = r[..., :-1]
    cy = torch.cat([torch.zeros_like(w_env[..., :1]), torch.cumsum(w_env.double(), -1)], -1)
    return torch.gather(cy, -1, hi) - torch.gather(cy, -1, lo)


def interlevel64(c, w, t_env, w_env, short=False):
    wo = outer64(c, t_env, w_env, short)
    w = w.double()
    return (torch.clip(w - wo, min=0) ** 2 / (w + EPS)).sum(-1) / w.shape[-1]


def interlevel_grad64(c, w, t_env, w_env, g):
    lo, hi = outer_ranges(c, t_env)
    wo = outer64(c, t_env, w_env)
    w = w.double()
    Nc, Np = w.shape[-1], w_env.shape[-1]
    dwo = -2 * torch.clip(w - wo, min=0) / (w + EPS) / Nc * g.double()[..., None]
    k = torch.arange(Np, device=w.device)
    inside = (lo[..., :, None] <= k) & (k < hi[..., :, None])                        # (n, Nc, Np)
    return (inside * dwo[..., None]).sum(-2)


def interlevel_bounds(c, w, t_env, w_env, g):
    """A-priori bounds: each w_outer_j carries len_j 2^-24 sum|w_env| (sequential sum); clip(w - w_outer)^2 / (w + eps) moves by at most
    2 delta_j per unit (c <= w); the per-ray sum and the /Nc add (Nc + 37) 2^-24 relative.  The gradient term -2c/(w + eps) moves by
    2 delta_j / (w_j + eps) + 4 2^-24 |term|, and each d w_env[k] sums at most Nc terms."""
    lo, hi = outer_ranges(c, t_env)
    w = w.double()
    we = w_env.double().abs()
    cy = torch.cat([torch.zeros_like(we[..., :1]), torch.cumsum(we, -1)], -1)
    S = torch.gather(cy, -1, hi) - torch.gather(cy, -1, lo)
    length = (hi - lo).double()
    delta = (length + 1) * U * S
    Nc, Np = w.shape[-1], w_env.shape[-1]
    wo = outer64(c, t_env, w_env)
    term = torch.clip(w - wo, min=0) ** 2 / (w + EPS)
    loss = (2 * delta + 4 * U * term).sum(-1) / Nc + (Nc + 37) * U * term.sum(-1) / Nc
    gj = (2 * delta / (w + EPS) + 8 * U * 2 * torch.clip(w - wo, min=0) / (w + EPS)) / Nc * g.double().abs()[..., None]
    dj = 2 * torch.clip(w - wo, min=0) / (w + EPS) / Nc * g.double().abs()[..., None]
    k = torch.arange(Np, device=w.device)
    inside = (lo[..., :, None] <= k) & (k < hi[..., :, None])
    grad = (inside * (gj + (Nc + 2) * U * dj)[..., None]).sum(-2)
    return loss, grad


# ---- bilinear upsampling, align_corners=True ----

def upsample_matrix(n_in: int, n_out: int, fp32: bool = True, short: bool = False) -> torch.Tensor:
    """(n_out, n_in) float64 matrix of one axis: ATen's h1r = scale * o, h1 = int(h1r), h1p = h1 < n_in - 1, lambda1 = h1r - h1.
    fp32: the weights as the kernel and ATen's fp32 forward compute them; else in float64.  `short` drops the last output row that reaches
    each input index (a mutant of the gather range)."""
    ft = np.float32 if fp32 else np.float64
    scale = ft(n_in - 1) / ft(n_out - 1) if n_out > 1 else ft(0)
    A = np.zeros((n_out, n_in))
    for o in range(n_out):
        r = ft(scale * ft(o))
        h1 = int(r)
        h1p = 1 if h1 < n_in - 1 else 0
        l1 = ft(r - ft(h1))
        l0 = ft(ft(1) - l1)
        A[o, h1] += float(l0)
        A[o, h1 + h1p] += float(l1)
    if short:
        for y in range(n_in):
            rows = np.nonzero(A[:, y])[0]
            if rows.size:
                A[rows[-1], y] = 0.0
    return torch.from_numpy(A)


def upsample64(x, size, fp32=True):
    Ah = upsample_matrix(x.shape[-2], size[0], fp32).to(x.device)
    Aw = upsample_matrix(x.shape[-1], size[1], fp32).to(x.device)
    return Ah @ x.double() @ Aw.T


def upsample_adjoint64(g, in_hw, fp32=True, short=False):
    Ah = upsample_matrix(in_hw[0], g.shape[-2], fp32, short).to(g.device)
    Aw = upsample_matrix(in_hw[1], g.shape[-1], fp32, short).to(g.device)
    return Ah.T @ g.double() @ Aw


def upsample_bound(g, in_hw):
    """The kernel sums, per input element, rows of <= n_x products and then <= n_y weighted rows: (n_x + n_y + 4) 2^-24 of
    sum |wy| |wx| |g|, with n_x, n_y <= 2 out / in + 2."""
    Ah = upsample_matrix(in_hw[0], g.shape[-2]).to(g.device)
    Aw = upsample_matrix(in_hw[1], g.shape[-1]).to(g.device)
    n = 2 * g.shape[-2] / in_hw[0] + 2 * g.shape[-1] / in_hw[1] + 8
    return n * U * (Ah.abs().T @ g.double().abs() @ Aw.abs())
