"""neo360_b200.bf16 derives every size, leading dimension and byte offset of the `neo_tc_*_bf16` calls from tensor views, and refuses
operands that do not agree before the library is called.  Runs on CPU tensors against a recorder standing in for the library."""
import pytest
import torch

from neo360_b200 import _lib as L
from neo360_b200 import bf16


class _Recorder:
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        return lambda *args: self.calls.append((name, args)) or 0


@pytest.fixture
def lib(monkeypatch):
    rec = _Recorder()
    monkeypatch.setattr(L, "load", lambda: rec)
    monkeypatch.setattr(L, "require_cuda", lambda t: None)
    return rec


def _bf(*shape):
    return torch.zeros(*shape, dtype=torch.bfloat16)


def test_gemm_column_block(lib):
    A, W, C = _bf(64, 1536), _bf(64, 512), _bf(64, 64)
    bf16.gemm(A[:, 512:1024], W, None, C, 1, None)
    (name, a), = lib.calls
    assert name == "neo_tc_gemm_bf16"
    assert a[0] == A.data_ptr() + 1024 and a[1] == 1536            # A + 512 bf16 elements, lda of the whole buffer
    assert a[2:4] == (W.data_ptr(), 512) and a[5:7] == (C.data_ptr(), 64)
    assert a[7:11] == (64, 64, 512, 1)                              # M, N, K, epilogue


def test_pack_transposed_feature_columns(lib):
    """_MLPTrainTC's W0^T / skip-layer feature columns: the F feature columns at c0 of a (W, c0 + F) weight, transposed into the first F
    rows of a (Kf, W) buffer -> (rows W, cols_in F, ld_in c0 + F, cols_out F, ld_out W)."""
    Wd, F, Kf, c0 = 256, 90, 128, 256
    w = torch.zeros(Wd, c0 + F)
    wt = _bf(Kf, Wd)
    bf16.pack(w[:, c0:c0 + F], wt[:F], True, None)
    (name, a), = lib.calls
    assert name == "neo_tc_pack_bf16"
    assert a == (w.data_ptr() + 4 * c0, Wd, F, c0 + F, wt.data_ptr(), F, Wd, 1, None)


def test_wgrad_k_valid(lib):
    dY, X, ws = _bf(128, 64), _bf(128, 576), torch.zeros(16, dtype=torch.uint8)
    dW = torch.zeros(64, 518)
    bf16.wgrad(dY, X, dW, None, ws, None)
    (name, a), = lib.calls
    assert name == "neo_tc_wgrad_bf16"
    assert a[4:7] == (128, 64, 576) and a[8] == 518                 # M, N, K, k_valid = dW.shape[1]


def test_refusals(lib):
    A, W, C = _bf(64, 512), _bf(64, 512), _bf(64, 64)
    with pytest.raises(ValueError):
        bf16.gemm(A, _bf(64, 576), None, C, 0, None)               # K mismatch
    with pytest.raises(ValueError):
        bf16.gemm(A.float(), W, None, C, 0, None)                  # fp32 where bf16 is required
    with pytest.raises(ValueError):
        bf16.gemm(_bf(512, 64).t(), W, None, C, 0, None)           # stride(-1) != 1
    with pytest.raises(ValueError):
        bf16.pack(torch.zeros(64, 32).t(), _bf(32, 64), False, None)
    assert lib.calls == []
