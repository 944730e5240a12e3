"""CPU: the SSIM model (oracle/metrics_model.py), the output-side golden vectors of the reference (tests/golden/metrics_reference_vectors.npz,
oracle/make_golden_metrics.py) and the argument checks of the new entry points."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch
from scipy import signal

from oracle import metrics_model as mm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(ROOT, "tests", "golden", "metrics_reference_vectors.npz"))


def ssim_2d(x: np.ndarray, y: np.ndarray) -> np.ndarray:
    """Independent restatement: the non-separable 11x11 window, scipy correlate2d "valid", one channel at a time."""
    g = mm.window_exact().numpy()
    w = np.outer(g, g)
    x, y = np.clip(x, 0, 1), np.clip(y, 0, 1)
    out = []
    for c in range(3):
        f = lambda v: signal.correlate2d(v[..., c], w, "valid")
        mx, my = f(x), f(y)
        sxx, syy, sxy = f(x * x) - mx * mx, f(y * y) - my * my, f(x * y) - mx * my
        out.append((2 * mx * my + mm.C1) / (mx * mx + my * my + mm.C1) * (2 * sxy + mm.C2) / (sxx + syy + mm.C2))
    return np.stack(out, -1)


@pytest.mark.parametrize("H,W", [(11, 11), (11, 40), (37, 53), (64, 64)])
def test_model_equals_2d_correlation(H, W):
    """1e-12, plus float64's own rounding of the cancellation G*(x x) - mu^2 where 1/(s_xx + s_yy + C2) amplifies it: the model's
    magnitude unit taken at 2^-53 instead of 2^-24 (nearly flat frames near 1 reach 1.5e-12)."""
    for k, fam in enumerate(mm.FAMILIES):
        x, y = mm.frames(fam, 2, H, W, seed=k)
        ss, mean = mm.ssim_f64(x, y)
        tol = 1e-12 + 8 * 2.0 ** -29 * mm.bound_unit(x, y).numpy()
        assert ss.shape == (2, H - 10, W - 10, 3)
        for i in range(2):
            ref = ssim_2d(x[i].double().numpy(), y[i].double().numpy())
            assert (np.abs(ss[i].numpy() - ref) <= tol[i]).all(), fam
            assert abs(float(mean[i]) - ref.mean()) <= tol[i].mean(), fam


def test_model_identity_and_symmetry():
    for k, fam in enumerate(mm.FAMILIES):
        x, y = mm.frames(fam, 2, 23, 31, seed=k)
        assert torch.equal(mm.ssim_f64(x, x)[0], torch.ones(2, 13, 21, 3, dtype=torch.float64)), fam
        assert (mm.ssim_f64(x, y)[0] - mm.ssim_f64(y, x)[0]).abs().max() <= 1e-15, fam


def test_window_constants_are_the_fp32_construction():
    """csrc/metrics.cu's window constants are torch's fp32 values of piqa's construction, and its C1 / C2 are float(0.01 ** 2) and
    float(0.03 ** 2); the float64 window differs from them only by fp32 rounding."""
    src = open(os.path.join(ROOT, "neo360_b200", "csrc", "metrics.cu")).read()
    body = re.search(r"c_win\[kTaps\] = \{([^}]*)\}", src).group(1)
    consts = [float.fromhex(v.strip().rstrip("f")) for v in body.split(",")]
    assert consts == mm.window_f32().tolist()
    assert np.abs(np.array(consts) - mm.window_exact().numpy()).max() <= 2 ** -24
    c1, c2 = re.search(r"kC1 = ([0-9.e-]+)f, kC2 = ([0-9.e-]+)f", src).groups()
    assert np.float32(c1) == np.float32(mm.C1) and np.float32(c2) == np.float32(mm.C2)


@pytest.mark.parametrize("H,W,n", [(11, 11, 3), (37, 53, 3), (120, 160, 2)])
def test_framework_form_within_bound(H, W, n):
    worst = 0.0
    for k, fam in enumerate(mm.FAMILIES):
        x, y = mm.frames(fam, n, H, W, seed=100 + k)
        ref, mref = mm.ssim_f64(x, y)
        unit = mm.bound_unit(x, y)
        got, mgot = mm.ssim_framework(x, y)
        r = float(((got.double() - ref).abs() / unit).max())
        worst = max(worst, r)
        assert r <= mm.BOUND_K, (fam, r)
        assert ((mgot.double() - mref).abs() <= mm.BOUND_K * unit.flatten(1).mean(-1)).all(), fam
    print(f"framework fp32 form: largest error {worst:.2f} units (bound {mm.BOUND_K})")


# ------------------------------------------------------------------------------------------------ reference golden vectors

def test_object_psnr_semantics_match_reference(gold):
    """psnr_obj_each's reduction (sum and count of the clipped squared errors over the masked pixels' values), restated in float64, is
    the reference's get_obj_rgbs_from_segmap + psnr_each within fp32 rounding; the empty mask gives NaN, the one-pixel mask a finite value."""
    preds, gts, masks = (torch.from_numpy(gold[k]) for k in ("preds", "gts", "masks"))
    got = []
    for p, g, m in zip(preds, gts, masks):
        d = (p.double().clamp(0, 1) - g.double().clamp(0, 1))[m]
        got.append(-10 * np.log10(float((d * d).sum()) / d.numel()) if d.numel() else float("nan"))
    got, ref = np.array(got), gold["psnr_obj"].astype(np.float64)
    assert np.isnan(ref[1]) and np.isnan(got[1])
    ok = ~np.isnan(ref)
    assert np.abs(got[ok] - ref[ok]).max() <= 1e-5 * np.abs(ref[ok]).max()


def test_depth_images_bit_for_bit(gold):
    pytest.importorskip("cv2")
    from neo360_b200 import output
    for key in ("rand", "const"):
        depths = list(torch.from_numpy(gold[f"depth_{key}"]))
        got = np.stack(output.depth_images(depths))
        assert got.dtype == np.uint8 and np.array_equal(got, gold[f"depth_img_{key}"]), key


def test_store_depth_img_writes_reference_arrays(gold, tmp_path, monkeypatch):
    pytest.importorskip("cv2")
    from PIL import Image
    from neo360_b200 import output
    seen = []
    orig = Image.fromarray
    monkeypatch.setattr(Image, "fromarray", lambda a, *x, **k: (seen.append(np.array(a, copy=True)), orig(a, *x, **k))[1])
    paths = output.store_depth_img(str(tmp_path), list(torch.from_numpy(gold["depth_rand"])), "depth_img")
    assert [os.path.basename(p) for p in paths] == [f"depth_img{i:03d}.jpg" for i in range(len(paths))]
    assert all(os.path.getsize(p) > 0 for p in paths)
    assert np.array_equal(np.stack(seen), gold["depth_img_rand"])


def test_store_depth_img_without_cv2_raises_clearly(monkeypatch):
    import builtins
    from neo360_b200 import output
    real = builtins.__import__
    monkeypatch.setattr(builtins, "__import__", lambda name, *a, **k: (_ for _ in ()).throw(ImportError(name)) if name == "cv2"
                        else real(name, *a, **k))
    with pytest.raises(RuntimeError, match="cv2"):
        output.depth_images([torch.zeros(2, 2)])


@pytest.mark.parametrize("case", ["neo360", "mip360"])
def test_write_stats_byte_equal(gold, tmp_path, case):
    from oracle.make_golden_metrics import STATS
    from neo360_b200 import output
    path = tmp_path / "results.json"
    output.write_stats(str(path), *STATS[case])
    assert path.read_bytes() == gold[f"stats_{case}"].tobytes()
    if case == "mip360":      # the object PSNR, passed last under the same name, is what results.json keeps under "PSNR"
        assert b"18.765432109876" in path.read_bytes() and b"25.0" not in path.read_bytes()


def test_stat_builder():
    from neo360_b200 import output
    v = torch.tensor([20.0, 22.0, 27.0])
    assert output.stat("PSNR", v) == {"name": "PSNR", "mean": 23.0, "test": 23.0}


def test_metrics_raise_on_cpu_tensors():
    from neo360_b200 import output
    x = torch.rand(16, 16, 3)
    with pytest.raises(RuntimeError, match="CUDA"):
        output.ssim(x, x)
    with pytest.raises(RuntimeError, match="CUDA"):
        output.ssim_each([x], [x])
    with pytest.raises(RuntimeError, match="CUDA"):
        output.psnr_obj_each([x], [x], [torch.ones(16, 16, dtype=torch.bool)])


# ------------------------------------------------------------------------------------------------ argument checks

@pytest.fixture(scope="module")
def lib():
    from neo360_b200 import build, _lib
    build.build()
    return _lib.load()


def test_ssim_argument_validation_without_gpu(lib):
    """`neo_ssim` rejects NULL buffers, n < 1, H or W < 11, sizes past int64 elements or 2^31 - 1 tiles and a short workspace before any
    launch (the pointers are never dereferenced); `neo_ssim_workspace_bytes` is 0 for the same sizes."""
    p = 1 << 20
    ws = lib.neo_ssim_workspace_bytes(2, 11, 11)
    assert ws == 2 * 8 and lib.neo_ssim_workspace_bytes(3, 480, 640) == 3 * 30 * 20 * 8
    call = lambda a, b, n, H, W, out, ssm, w, nb: lib.neo_ssim(a, b, n, H, W, out, ssm, w, nb, None)
    for args in ((None, p, 2, 11, 11, p, p, p, ws), (p, None, 2, 11, 11, p, None, p, ws), (p, p, 2, 11, 11, None, p, p, ws),
                 (p, p, 2, 11, 11, p, p, None, ws), (p, p, 0, 11, 11, p, p, p, ws), (p, p, -1, 11, 11, p, p, p, ws),
                 (p, p, 2, 10, 11, p, p, p, ws), (p, p, 2, 11, 10, p, p, p, ws), (p, p, 2, 11, 0, p, p, p, ws),
                 (p, p, 1 << 30, 1 << 30, 1 << 30, p, p, p, 1 << 62), (p, p, 1 << 20, 1 << 16, 1 << 16, p, p, p, 1 << 62)):
        assert call(*args) == -1, args
        assert b"neo_ssim" in lib.neo_last_error()
    assert call(p, p, 2, 11, 11, p, None, p, ws - 1) == -3
    assert call(p, p, 2, 11, 11, p, None, p + 4, ws) == -3
    for n, H, W in ((0, 11, 11), (1, 10, 11), (1, 11, 10), (1 << 30, 1 << 30, 1 << 30), (1 << 20, 1 << 16, 1 << 16)):
        assert lib.neo_ssim_workspace_bytes(n, H, W) == 0


def test_masked_sq_err_argument_validation_without_gpu(lib):
    p = 1 << 20
    call = lambda a, b, m, n, s, c: lib.neo_clipped_sq_err_masked(a, b, m, n, s, c, None)
    for args in ((None, p, p, 5, p, p), (p, None, p, 5, p, p), (p, p, None, 5, p, p), (p, p, p, 5, None, p), (p, p, p, 5, p, None),
                 (p, p, p, 0, p, p), (p, p, p, -3, p, p), (p, p, p, (1 << 61) + 1, p, p)):
        assert call(*args) == -1, args
        assert b"neo_clipped_sq_err_masked" in lib.neo_last_error()
    assert lib.neo_clipped_sq_err(p, p, C.c_longlong(0), p, None) == -1
