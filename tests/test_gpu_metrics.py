"""GPU: the output-side metrics of neo360_b200.output against oracle/metrics_model.py and the reference's golden vectors.

* `neo_ssim`: the ss map per pixel and each frame's mean within BOUND_K magnitude units of the float64 model (bound_unit), at 11x11 (one
  output pixel), 11x12, 12x11, 37x53, 480x640 and 960x1280 with n = 1, 3 and 100, every frame of a batch a different content family
  (uniform noise, box-filtered, constant, nearly flat near 0.5 and near 1, out of range, black against white, identical); map entries
  the kernel does not write keep a NaN sentinel and fail.  SSIM(x, x) is exactly 1.  Two calls are bit-identical, and a frame alone
  gives the bits it gets inside a batch of 100.
* `psnr_obj_each`: float64 of the masked clipped squared error, NaN for an empty mask, the reference's values on the golden frames.
* `neo_clipped_sq_err` (psnr / psnr_each) keeps its values.

Run with `-m gpu -s` to see the measured fraction of each bound.
"""
import os

import numpy as np
import pytest
import torch

from oracle import metrics_model as mm

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORST = {}
CASES = [(11, 11, 1), (11, 11, 3), (11, 12, 3), (12, 11, 3), (37, 53, 1), (37, 53, 3), (37, 53, 100), (480, 640, 3), (480, 640, 100),
         (960, 1280, 1), (960, 1280, 100)]


@pytest.fixture(scope="module")
def cuda():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from neo360_b200 import build
    build.build()
    return torch.device("cuda:0")


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    print("\nmeasured (largest over all cases): " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(WORST.items())))


def note(key, v):
    WORST[key] = max(WORST.get(key, 0.0), float(v))


def batch(n, H, W, seed, dev):
    """n frames, frame i of family FAMILIES[(i + seed) % 8], each seeded on its own."""
    xs, ys = zip(*(mm.frames(mm.FAMILIES[(i + seed) % len(mm.FAMILIES)], 1, H, W, seed=1000 * seed + i) for i in range(n)))
    return torch.cat(xs).to(dev), torch.cat(ys).to(dev)


def run_ssim(x, y):
    """neo_ssim with a NaN-filled map: (per-frame float64 values, fp32 map)."""
    from neo360_b200 import _lib as L
    n, H, W, _ = x.shape
    lib = L.load()
    nb = lib.neo_ssim_workspace_bytes(n, H, W)
    ws = torch.full((nb // 8,), float("nan"), dtype=torch.float64, device=x.device)
    out = torch.full((n,), float("nan"), dtype=torch.float64, device=x.device)
    ss = torch.full((n, H - 10, W - 10, 3), float("nan"), dtype=torch.float32, device=x.device)
    L.check(lib.neo_ssim(x.data_ptr(), y.data_ptr(), n, H, W, out.data_ptr(), ss.data_ptr(), ws.data_ptr(), nb,
                         torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return out, ss


@pytest.mark.parametrize("H,W,n", CASES)
def test_ssim_vs_float64_model(cuda, H, W, n):
    x, y = batch(n, H, W, seed=H + W + n, dev=cuda)
    got, ss = run_ssim(x, y)
    for i in range(n):
        ref, mref = mm.ssim_f64(x[i], y[i])
        unit = mm.bound_unit(x[i], y[i])
        r = float(((ss[i].double() - ref).abs() / unit).max())        # NaN (an unwritten entry) fails the comparison below
        assert r <= mm.BOUND_K, (i, mm.FAMILIES[(i + H + W + n) % len(mm.FAMILIES)], r)
        note("map", r)
        rm = abs(float(got[i]) - float(mref)) / float(unit.mean())
        assert rm <= mm.BOUND_K, (i, rm)
        note("mean", rm)
    # the per-frame value is the mean of the kernel's own map
    assert torch.allclose(got, ss.double().flatten(1).mean(-1), rtol=0, atol=1e-12)


@pytest.mark.parametrize("H,W", [(11, 11), (37, 53), (480, 640)])
def test_ssim_of_identical_frames_is_exactly_one(cuda, H, W):
    xs = [mm.frames(f, 1, H, W, seed=k)[0] for k, f in enumerate(mm.FAMILIES)]
    x = torch.cat(xs).to(cuda)
    got, ss = run_ssim(x, x.clone())
    assert (ss == 1.0).all() and (got == 1.0).all()


@pytest.mark.parametrize("H,W", [(37, 53), (480, 640)])
def test_ssim_deterministic_and_batch_invariant(cuda, H, W):
    x, y = batch(100, H, W, seed=7, dev=cuda)
    a, sa = run_ssim(x, y)
    b, sb = run_ssim(x, y)
    assert torch.equal(a, b) and torch.equal(sa, sb)
    for k in (0, 1, 37, 99):
        c, sc = run_ssim(x[k:k + 1].contiguous(), y[k:k + 1].contiguous())
        assert torch.equal(c[0], a[k]) and torch.equal(sc[0], sa[k]), k


def test_ssim_python_api(cuda):
    from neo360_b200 import output
    x, y = batch(5, 40, 52, seed=3, dev=cuda)
    u, v = batch(2, 23, 17, seed=4, dev=cuda)
    preds = [x[0], u[0], x[1], x[2], u[1], x[3], x[4]]
    gts = [y[0], v[0], y[1], y[2], v[1], y[3], y[4]]
    vals = output.ssim_each(preds, gts)
    assert vals.dtype == torch.float32 and vals.shape == (7,)
    singles = torch.tensor([output.ssim(p, g) for p, g in zip(preds, gts)], dtype=torch.float64)
    assert torch.equal(vals, singles.float())
    full, ss = output.ssim_batch(x, y, return_map=True)
    assert torch.equal(full, run_ssim(x, y)[0]) and torch.equal(ss, run_ssim(x, y)[1])
    for i, j in enumerate((0, 2, 3, 5, 6)):
        assert float(vals[j]) == float(np.float32(full[i].item()))
    with pytest.raises(ValueError):
        output.ssim_batch(x[:, :10], y[:, :10])


def test_psnr_obj_each_vs_float64(cuda):
    from neo360_b200 import output
    g = torch.Generator().manual_seed(3)
    H, W = 96, 128
    preds = (1.4 * torch.rand(6, H, W, 3, generator=g) - 0.2).to(cuda)
    gts = (1.4 * torch.rand(6, H, W, 3, generator=g) - 0.2).to(cuda)
    masks = (torch.rand(6, H, W, generator=g) < 0.25).to(cuda)
    masks[1] = False
    masks[2] = False
    masks[2, 50, 3] = True
    masks[3] = True
    m_u8 = masks.to(torch.uint8) * 7                 # any non-zero byte selects
    for mk in (masks, m_u8):
        got = output.psnr_obj_each(list(preds), list(gts), list(mk))
        for i in range(6):
            sel = mk[i] != 0
            d = (preds[i].double().clamp(0, 1) - gts[i].double().clamp(0, 1))[sel]
            if d.numel() == 0:
                assert np.isnan(float(got[i]))
                continue
            ref = -10 * np.log10(float((d * d).sum()) / d.numel())
            assert abs(float(got[i]) - ref) <= 1e-5 * abs(ref), i
    full = output.psnr_each(list(preds), list(gts))
    assert abs(float(got[3]) - float(full[3])) <= 1e-5 * abs(float(full[3]))


def test_psnr_and_object_psnr_match_reference_golden(cuda):
    from neo360_b200 import output
    gold = np.load(os.path.join(ROOT, "tests", "golden", "metrics_reference_vectors.npz"))
    preds, gts = torch.from_numpy(gold["preds"]).to(cuda), torch.from_numpy(gold["gts"]).to(cuda)
    masks = torch.from_numpy(gold["masks"]).to(cuda)
    obj = output.psnr_obj_each(list(preds), list(gts), list(masks)).numpy()
    ref = gold["psnr_obj"]
    assert np.array_equal(np.isnan(obj), np.isnan(ref)) and np.isnan(ref[1])
    ok = ~np.isnan(ref)
    assert np.abs(obj[ok] - ref[ok]).max() <= 4e-6 * np.abs(ref[ok]).max()
    ps = output.psnr_each(list(preds), list(gts)).numpy()
    assert np.abs(ps - gold["psnr"]).max() <= 4e-6 * np.abs(gold["psnr"]).max()


def test_clipped_sq_err_keeps_its_values(cuda):
    """neo_clipped_sq_err: the float64 sum of the fp32 squared clipped differences, as before the masked form shared its kernel."""
    from neo360_b200 import _lib as L
    g = torch.Generator().manual_seed(9)
    for n in (1, 255, 256, 257, 100_003, 3 * 480 * 640):
        a = (1.4 * torch.rand(n, generator=g) - 0.2).to(cuda)
        b = (1.4 * torch.rand(n, generator=g) - 0.2).to(cuda)
        out = torch.zeros(1, dtype=torch.float64, device=cuda)
        L.check(L.load().neo_clipped_sq_err(a.data_ptr(), b.data_ptr(), n, out.data_ptr(), torch.cuda.current_stream().cuda_stream))
        d = a.clamp(0, 1) - b.clamp(0, 1)
        ref = float((d * d).double().sum())
        assert abs(float(out) - ref) <= 1e-12 * max(ref, 1e-30), n
