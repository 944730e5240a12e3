"""TEST INFRASTRUCTURE ONLY.  Float64 model of the SSIM that LitModel.ssim_each computes with piqa's SSIM() at its defaults
(models/interface.py:101-111), an a-priori per-pixel error bound for an fp32 evaluation of it, and the fp32 framework form.

piqa is not installed here, so the definition is pinned as csrc/metrics.cu states it: inputs clipped to [0, 1]; an 11-tap Gaussian window,
sigma 1.5, applied separably without padding (the map of an (H, W) channel is (H-10, W-10)); mu_x = G*x, s_xx = G*(x x) - mu_x^2 (and y,
xy alike); C1 = 0.01^2, C2 = 0.03^2; cs = (2 s_xy + C2) / (s_xx + s_yy + C2); ss = (2 mu_x mu_y + C1) / (mu_x^2 + mu_y^2 + C1) * cs; a
frame's SSIM is the mean of ss over its three channels and every valid pixel.

* `ssim_f64`: the float64 model with the exact Gaussian weights, on (..., H, W, 3) frames of any device; map (..., H-10, W-10, 3) and the
  per-frame mean.
* `bound_unit`: the per-pixel magnitude unit of an fp32 evaluation.  Each of G*(x x), G*(y y), G*(x y) is a sum of non-negative (or, for
  x y, signed) terms, so its fp32 error is a few 2^-24 (G*x x + G*y y + 2 |G*x y|); s = G*(x x) - mu^2 keeps that absolute error while
  it cancels, and cs divides it by s_xx + s_yy + C2 (C2 is only 9e-4).  The luminance factor and the three divisions add a few 2^-24
  relative, and |cs|, |luminance| <= 1.  Unit = 2^-24 ((G*x x + G*y y + 2 |G*x y|) / (s_xx + s_yy + C2) + 1); an fp32 evaluation is
  within BOUND_K units of the model per pixel (BOUND_K is 2-3x the largest value measured, DESIGN.md section 2).
* `ssim_framework`: what piqa runs, in the framework's fp32: torch conv2d with the fp32 window built as piqa builds it, on (n, 3, H, W).
* `frames`: the seeded test content shared by the CPU and GPU tests.
"""
import numpy as np
import torch
import torch.nn.functional as F

TAPS, SIGMA = 11, 1.5
C1, C2 = 0.01 ** 2, 0.03 ** 2
U = 2.0 ** -24
BOUND_K = 16.0        # measured: neo_ssim 5.49 (H100 80GB HBM3, 700 W), fp32 framework form on the CPU 4.5

FAMILIES = ("noise", "smooth", "constant", "flat", "flat_bright", "out_of_range", "black_white", "identical")


def window_exact() -> torch.Tensor:
    i = torch.arange(TAPS, dtype=torch.float64) - (TAPS - 1) / 2
    k = torch.exp(-(i ** 2) / (2 * SIGMA ** 2))
    return k / k.sum()


def window_f32() -> torch.Tensor:
    """piqa's gaussian_kernel(11, 1.5), step by step in fp32."""
    k = torch.arange(TAPS, dtype=torch.float)
    k -= (TAPS - 1) / 2
    k = k ** 2 / (2. * SIGMA ** 2)
    k = torch.exp(-k)
    k /= k.sum()
    return k


def _filter(v: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """Valid separable filter of (..., H, W, C) along W and then H."""
    K = w.numel()
    Wo, Ho = v.shape[-2] - K + 1, v.shape[-3] - K + 1
    h = sum(w[k] * v[..., :, k:k + Wo, :] for k in range(K))
    return sum(w[k] * h[..., k:k + Ho, :, :] for k in range(K))


def moments(x: torch.Tensor, y: torch.Tensor):
    """mu_x, mu_y, G*(x x), G*(y y), G*(x y) in float64 of the clipped frames (..., H, W, 3)."""
    x = x.double().clamp(0, 1)
    y = y.double().clamp(0, 1)
    w = window_exact().to(x.device)
    return _filter(x, w), _filter(y, w), _filter(x * x, w), _filter(y * y, w), _filter(x * y, w)


def ssim_f64(x: torch.Tensor, y: torch.Tensor):
    """(ss map (..., H-10, W-10, 3), per-frame mean (...)) in float64."""
    mx, my, gxx, gyy, gxy = moments(x, y)
    sxx, syy, sxy = gxx - mx * mx, gyy - my * my, gxy - mx * my
    cs = (2 * sxy + C2) / (sxx + syy + C2)
    ss = (2 * mx * my + C1) / (mx * mx + my * my + C1) * cs
    return ss, ss.flatten(-3).mean(-1)


def bound_unit(x: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
    """Per-pixel magnitude unit (module docstring), same shape as the map."""
    mx, my, gxx, gyy, gxy = moments(x, y)
    den = (gxx - mx * mx) + (gyy - my * my) + C2
    return U * ((gxx + gyy + 2 * gxy.abs()) / den + 1)


def ssim_framework(x: torch.Tensor, y: torch.Tensor):
    """fp32 framework form of (n, H, W, 3) frames: (map (n, H-10, W-10, 3), per-frame mean (n)), on the frames' device with the
    framework's default conv2d settings there (TF32 on an Ampere or later GPU unless torch.backends.cudnn.allow_tf32 is off)."""
    x = x.float().clamp(0, 1).permute(0, 3, 1, 2)
    y = y.float().clamp(0, 1).permute(0, 3, 1, 2)
    k = window_f32().to(x.device)
    kv, kh = k.view(1, 1, TAPS, 1).expand(3, 1, TAPS, 1), k.view(1, 1, 1, TAPS).expand(3, 1, 1, TAPS)

    def filt(v):
        return F.conv2d(F.conv2d(v, kv, groups=3), kh, groups=3)

    mx, my = filt(x), filt(y)
    mxx, myy, mxy = mx ** 2, my ** 2, mx * my
    sxx, syy, sxy = filt(x ** 2) - mxx, filt(y ** 2) - myy, filt(x * y) - mxy
    cs = (2 * sxy + C2) / (sxx + syy + C2)
    ss = (2 * mxy + C1) / (mxx + myy + C1) * cs
    ss = ss.permute(0, 2, 3, 1)
    return ss, ss.flatten(1).mean(-1)


def frames(family: str, n: int, H: int, W: int, seed: int = 0, device="cpu"):
    """Seeded fp32 (n, H, W, 3) pairs (pred, gt) of one content family."""
    g = torch.Generator().manual_seed(seed)
    r = lambda: torch.rand(n, H, W, 3, generator=g)
    if family == "noise":
        x, y = r(), r()
    elif family == "smooth":       # 7x7 box-filtered noise, correlated pair
        box = lambda v: F.avg_pool2d(v.permute(0, 3, 1, 2), 7, 1, 3, count_include_pad=False).permute(0, 2, 3, 1)
        x = box(r())
        y = box(0.7 * x + 0.3 * r())
    elif family == "constant":
        x = torch.rand(n, 1, 1, 3, generator=g).expand(n, H, W, 3).clone()
        y = torch.rand(n, 1, 1, 3, generator=g).expand(n, H, W, 3).clone()
    elif family == "flat":         # variances far below C2: the denominators approach C2
        x, y = 0.5 + 1e-3 * r(), 0.5 + 1e-3 * r()
    elif family == "flat_bright":  # the same near 1, where G*(x x) - mu^2 cancels the most
        x, y = 0.999 - 1e-3 * r(), 0.999 - 1e-3 * r()
    elif family == "out_of_range":
        x, y = 2 * r() - 0.5, 2 * r() - 0.5
    elif family == "black_white":
        x, y = torch.zeros(n, H, W, 3), torch.ones(n, H, W, 3)
    elif family == "identical":
        x = r()
        y = x.clone()
    else:
        raise ValueError(family)
    return x.contiguous().to(device), y.contiguous().to(device)
