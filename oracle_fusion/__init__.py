"""numpy oracle of the classifier's attention-weighted image-feature fusion -- TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and the benchmark scripts may import this package; deepi2p_b200.point_ops never
does.  It restates DESIGN.md 4.17 as explicit loops over the summed index in ascending order, vectorised over the
other two: one fp64 accumulator per output starting at +0.0, the float32 operands' products (exact in fp64) added one
at a time, the sum divided by P in fp64 and rounded once to float32.  No matmul or einsum: BLAS reorders the sums.

Each function returns float32 arrays; f64=True returns the fp64 quotients before the final rounding instead, and
with_abs=True also returns the fp64 sums of the terms' magnitudes divided by P (the scale of the error bound against
the reference's float32 arithmetic).
"""
import numpy as np


def _f64(a):
    return np.asarray(a, dtype=np.float32).astype(np.float64)


def _finish(S, T, P, f64, with_abs):
    with np.errstate(over="ignore", invalid="ignore"):
        q = S / np.float64(P)
        out = q if f64 else q.astype(np.float32)
    return (out, T / np.float64(P)) if with_abs else out


def forward(img_features, attention, f64=False, with_abs=False):
    """out [B,C,M] = float((sum over p ascending of F[b,c,p] * A[b,p,m]) / P)."""
    F, A = _f64(img_features), _f64(attention)
    B, C, P = F.shape
    M = A.shape[2]
    S = np.zeros((B, C, M))
    T = np.zeros((B, C, M))
    with np.errstate(over="ignore", invalid="ignore"):
        for p in range(P):
            t = F[:, :, p, None] * A[:, p, None, :]
            S += t
            T += np.abs(t)
    return _finish(S, T, P, f64, with_abs)


def backward_features(attention, grad_out, f64=False, with_abs=False):
    """gF [B,C,P] = float((sum over m ascending of gO[b,c,m] * A[b,p,m]) / P)."""
    A, G = _f64(attention), _f64(grad_out)
    B, P, M = A.shape
    C = G.shape[1]
    S = np.zeros((B, C, P))
    T = np.zeros((B, C, P))
    with np.errstate(over="ignore", invalid="ignore"):
        for m in range(M):
            t = G[:, :, m, None] * A[:, None, :, m]
            S += t
            T += np.abs(t)
    return _finish(S, T, P, f64, with_abs)


def backward_attention(img_features, grad_out, f64=False, with_abs=False):
    """gA [B,P,M] = float((sum over c ascending of F[b,c,p] * gO[b,c,m]) / P)."""
    F, G = _f64(img_features), _f64(grad_out)
    B, C, P = F.shape
    M = G.shape[2]
    S = np.zeros((B, P, M))
    T = np.zeros((B, P, M))
    with np.errstate(over="ignore", invalid="ignore"):
        for c in range(C):
            t = F[:, c, :, None] * G[:, c, None, :]
            S += t
            T += np.abs(t)
    return _finish(S, T, P, f64, with_abs)
