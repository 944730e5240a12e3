"""The bf16 tensor-core products of the training paths (`neo_tc_*_bf16`) on row views: 2-D views with contiguous rows, so a column block
is a slice such as `A[:, 512:1024]`.  M, N, K, k_valid and the leading dimensions come from shapes and `stride(0)`; a dtype or shape
that does not agree raises ValueError before the library is called."""
import torch

from . import _lib as L


def rows(t, dtype=torch.bfloat16):
    """(pointer, leading dimension in elements) of a row view of `dtype`."""
    if t.dtype != dtype or t.dim() != 2 or t.stride(-1) != 1:
        raise ValueError(f"expected a 2-D {dtype} view with contiguous rows, got {t.dtype} {tuple(t.shape)} strides {t.stride()}")
    L.require_cuda(t)
    return t.data_ptr(), t.stride(0)


def _vec(t, n):
    """pointer of an fp32 vector of n elements (None -> NULL)."""
    if t is not None and (t.dtype != torch.float32 or t.numel() != n):
        raise ValueError(f"expected {n} fp32 elements, got {t.dtype} {tuple(t.shape)}")
    return L.ptr(t)


def _agree(what, *shapes):
    for got, want in shapes:
        if tuple(got) != tuple(want):
            raise ValueError(f"{what}: shape {tuple(got)}, expected {tuple(want)}")


def pack(src, out, transpose, stream):
    """out = bf16(src), src an fp32 (rows, cols_in) view: out (rows, cols_out) zero past cols_in, or with `transpose` out (cols_out,
    rows) = the first cols_out columns of src transposed."""
    a, lda = rows(src, torch.float32)
    c, ldc = rows(out)
    r, k = src.shape
    cols = out.shape[0] if transpose else out.shape[1]
    _agree("pack out", (out.shape, (cols, r) if transpose else (r, cols)))
    if transpose and cols > k:
        raise ValueError(f"pack: {cols} columns transposed out of {k}")
    L.check(L.load().neo_tc_pack_bf16(a, r, k, lda, c, cols, ldc, int(transpose), stream))


def gemm(A, W, bias, C, epilogue, stream):
    """C (M,N) = A (M,K) . W (N,K)^T + bias (N or None), epilogue 0 = ReLU -> bf16, 1 -> bf16, 2 -> fp32."""
    a, lda = rows(A)
    w, ldw = rows(W)
    c, ldc = rows(C, torch.float32 if epilogue == 2 else torch.bfloat16)
    (M, K), N = A.shape, W.shape[0]
    _agree("gemm W, C", (W.shape, (N, K)), (C.shape, (M, N)))
    L.check(L.load().neo_tc_gemm_bf16(a, lda, w, ldw, _vec(bias, N), c, ldc, M, N, K, epilogue, stream))


def dgrad(dY, Wt, X, g_sig, w_sig, dX, stream):
    """dX (M,N) = (dY (M,K) . Wt (N,K)^T + g_sig (M) w_sig (N)^T) [X (M,N) > 0]; X None: no mask; g_sig, w_sig both or neither."""
    y, ldy = rows(dY)
    wt, ldwt = rows(Wt)
    dx, lddx = rows(dX)
    (M, K), N = dY.shape, Wt.shape[0]
    x, ldx = (None, 0) if X is None else rows(X)
    _agree("dgrad Wt, dX, X", (Wt.shape, (N, K)), (dX.shape, (M, N)), (dX.shape if X is None else X.shape, (M, N)))
    L.check(L.load().neo_tc_dgrad_bf16(y, ldy, wt, ldwt, x, ldx, _vec(g_sig, M), _vec(w_sig, N), dx, lddx, M, N, K, stream))


def wgrad(dY, X, dW, db, ws, stream):
    """dW (N, k_valid) fp32 = dY (M,N)^T X (M,K) without the columns past k_valid, db (N) = column sums of dY or None; `ws` is a
    workspace of neo_tc_wgrad_bf16_workspace_bytes(M, N, K) bytes or more."""
    y, ldy = rows(dY)
    x, ldx = rows(X)
    (M, N), K = dY.shape, X.shape[1]
    _agree("wgrad X", (X.shape, (M, K)))
    if dW.dtype != torch.float32 or dW.dim() != 2 or dW.shape[0] != N or dW.shape[1] > K:
        raise ValueError(f"wgrad dW: {dW.dtype} {tuple(dW.shape)}, expected fp32 ({N}, <= {K})")
    L.check(L.load().neo_tc_wgrad_bf16(y, ldy, x, ldx, M, N, K, L.ptr(dW), dW.shape[1], _vec(db, N), L.ptr(ws), ws.numel(), stream))


def relu_rank1(g, w, X, out, stream):
    """out (M,N) bf16 = (g (M) w (N)^T) [X (M,N) > 0]."""
    x, ldx = rows(X)
    o, ldo = rows(out)
    M, N = X.shape
    _agree("relu_rank1 out", (out.shape, (M, N)))
    L.check(L.load().neo_tc_relu_rank1_bf16(_vec(g, M), _vec(w, N), x, ldx, M, N, o, ldo, stream))


def rowdot(H, w, b, out, stream):
    """out (M, N) fp32 = H (M,K) . w (N,K)^T + b (N)."""
    h, ld = rows(H)
    (M, K), N = H.shape, w.shape[0]
    _agree("rowdot w", (w.shape, (N, K)))
    L.check(L.load().neo_tc_rowdot_bf16(h, ld, K, _vec(w, N * K), _vec(b, N), N, M, _vec(out, M * N), stream))
