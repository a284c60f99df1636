"""Exact integer cases for the fused TF32 kernels (test_tf32_exact_gpu.py) and their references, tested on their own.

An operand that is a small integer, or a dyadic value with at most 11 significant bits, is its own TF32 rounding; the
product of two of them is exact in float32; and while every partial sum is a multiple of the operands' finest step
below 2^24 of those steps, float32 accumulation is exact in any order.  A kernel's output must then equal a plain
reference bit for bit, whatever its tiling, split count or summation order, so a dropped, duplicated or misplaced
point, row or tap is a definite mismatch instead of an error under a TF32 tolerance.

The references come from the operations' definitions: float64 matrix products of integers (exact far below 2^53), a
float64 torch conv2d on the CPU, a brute-force lexsort for the kNN, and Fractions / mpmath for BatchNorm's statistics.
Every generator asserts its case's exactness preconditions and its sensitivity (no all-zero input row, point column,
weight column or conv tap, no channel that ReLU zeroes everywhere), so a case cannot silently become inexact or
blind."""
from fractions import Fraction

import mpmath
import numpy as np
import pytest
import torch

from oracle_pointwise import tf32_round

EXACT = 2.0 ** 24          # every partial sum, in units of the finest step, stays below this
AIM = 2.0 ** 20            # and the cases aim below this
REREAD = 2.0 ** 11         # a value a later layer re-reads (and rounds to TF32) stays below this

# point_chain.cu's constants
PC_TILE, DW_PTS, DW_TILE, DW_TARGET_CTAS, DW_MAX_SPLITS = 64, 32, 64, 1056, 256


# ---------------------------------------------------------------------------------------------------------------------
# preconditions


def assert_tf32(*arrays):
    """Every value is its own TF32 rounding (so the kernels' tf32_rna is the identity on it)."""
    for a in arrays:
        a = np.asarray(a, dtype=np.float32)
        assert np.array_equal(tf32_round(a), a), "an operand is not exactly representable in TF32"


def assert_steps(a, step):
    """Every value of a is an integer multiple of `step` (a power of two)."""
    a = np.asarray(a, dtype=np.float64)
    assert np.array_equal(np.round(a / step) * step, a), f"a value is not a multiple of {step}"


def assert_sum_bound(sum_abs, step=1.0, aim=True):
    """Sigma |terms| of every output element, in units of `step`, below 2^24 (and below 2^20 where the case aims)."""
    top = float(np.max(sum_abs)) / step
    assert top < EXACT, f"sum |terms| reaches {top:.3g} steps, not below 2^24"
    if aim:
        assert top <= AIM, f"sum |terms| reaches {top:.3g} steps, above the 2^20 the cases aim for"


def assert_reread(a):
    assert float(np.max(np.abs(a))) < REREAD, "an activation a later layer re-reads is not below 2^11"


def assert_no_zero_rows(a, axes, what):
    """No slice of `a` along the kept axes is all zero: reduce over `axes`."""
    assert np.all(np.any(np.asarray(a) != 0, axis=axes)), f"{what}: an all-zero slice"


def assert_relu_live(pre, axes):
    """No channel that ReLU zeroes everywhere: every channel has a positive pre-activation somewhere."""
    assert np.all(np.any(np.asarray(pre) > 0, axis=axes)), "a channel is zeroed by ReLU everywhere"


# ---------------------------------------------------------------------------------------------------------------------
# generators


def ints(rng, shape, amp):
    """float32 nonzero integers in [-amp, amp]."""
    v = rng.integers(1, amp + 1, size=shape) * rng.choice(np.array([-1, 1]), size=shape)
    return v.astype(np.float32)


def sparse_weights(rng, C_out, C_in, per_row, amp):
    """W [C_out, C_in]: integers in [-amp, amp], per_row nonzeros per row at random columns, and every input column j
    also feeding row j % C_out, so no row and no column is all zero."""
    W = np.zeros((C_out, C_in), dtype=np.float32)
    for c in range(C_out):
        cols = rng.choice(C_in, size=min(per_row, C_in), replace=False)
        W[c, cols] = ints(rng, len(cols), amp)
    j = np.arange(C_in)
    W[j % C_out, j] = ints(rng, C_in, amp)
    assert_no_zero_rows(W, 1, "weight row")
    assert_no_zero_rows(W, 0, "weight column")
    return W


def split_rows(K, n_src):
    """Source widths of K rows for n_src sources: with three or more, one boundary on the 64-row chunk edge where K
    allows, the others inside a chunk."""
    if n_src == 1 or K < n_src:
        return [K]
    on = [64] if K > 64 and n_src >= 3 else []
    inside = [int(c) + (int(c) % 64 == 0) for c in np.linspace(0, K, n_src - len(on) + 1)[1:-1]]
    cuts = sorted({c for c in on + inside if 0 < c < K})
    bounds = [0] + cuts + [K]
    return [b - a for a, b in zip(bounds, bounds[1:])]


def dw_splits(B, N, C, K):
    """point_chain_dw_f32's split count: about 1056 CTAs over the 64 x 64 tiles of dW, at most 256 and at most the
    number Q of 32-point chunks."""
    tiles = -(-C // DW_TILE) * -(-K // DW_TILE)
    Q = B * -(-N // DW_PTS)
    return max(1, min(-(-DW_TARGET_CTAS // tiles), DW_MAX_SPLITS, Q))


def chain_case(rng, B, N, c_in, widths, relus, amp_x=2, per_row=None, amp_w=1, x=None):
    """A dense chain of integer layers over x [B, c_in, N] (drawn when not given): (x, layers [(W, b, relu)], the
    exact output, the pre-activations).  Layer 1 is dense (or per_row-sparse), later layers are sparse selections;
    asserts every precondition on x itself."""
    x = ints(rng, (B, c_in, N), amp_x) if x is None else np.asarray(x, dtype=np.float32)
    layers, a, pres = [], x.astype(np.float64), []
    k = c_in
    for l, (C, relu) in enumerate(zip(widths, relus)):
        if l == 0:
            W = sparse_weights(rng, C, k, per_row, amp_w) if per_row is not None else ints(rng, (C, k), amp_w)
        else:                                  # a sparse selection of the (non-negative) previous activations
            W = np.abs(sparse_weights(rng, C, k, 2, amp_w))
        b = rng.integers(-3, 4, size=C).astype(np.float32)
        pre = mm(W, a) + b[None, :, None]
        if relu:                               # raise the bias of a channel ReLU would zero everywhere
            top = pre.max(axis=(0, 2))
            b = np.where(top > 0, b, b + 1 - top).astype(np.float32)
            pre = mm(W, a) + b[None, :, None]
        assert_tf32(W, b, a)
        assert_sum_bound(mm(np.abs(W), np.abs(a)) + np.abs(b)[None, :, None])
        if relu:
            assert_relu_live(pre, (0, 2))
        pres.append(pre)
        a = np.maximum(pre, 0.0) if relu else pre
        if l < len(widths) - 1:
            assert_reread(a)
        layers.append((W, b, relu))
        k = C
    assert_no_zero_rows(x, (0, 2), "input row")
    assert_no_zero_rows(x, 1, "point column")
    return x, layers, a, pres


# ---------------------------------------------------------------------------------------------------------------------
# references


def mm(W, x):
    """W [C, K] . x [B, K, N] in float64: exact for the integer and dyadic cases here (far below 2^53)."""
    return np.matmul(np.asarray(W, dtype=np.float64)[None], np.asarray(x, dtype=np.float64))


def ref_dw(dy, x):
    """dW [C, K] = sum over b, n of dy [B, C, N] x [B, K, N]^T, and db [C], in float64."""
    dy, x = np.asarray(dy, dtype=np.float64), np.asarray(x, dtype=np.float64)
    return np.einsum("bcn,bkn->ck", dy, x, optimize=True), dy.sum(axis=(0, 2))


def ref_partials(v, w=None):
    """The stats epilogue's per-(sample, 64-point tile, channel) sums: [B, ntiles, 2, C] float64 of (sum v, sum v^2),
    or of (sum v, sum w) for the act-grad epilogue; points past N count as zero."""
    v = np.asarray(v, dtype=np.float64)
    B, C, N = v.shape
    T = -(-N // PC_TILE)
    pad = lambda a: np.concatenate([a, np.zeros((B, C, T * PC_TILE - N))], axis=2).reshape(B, C, T, PC_TILE)
    s = pad(v).sum(axis=3)
    q = (pad(v) ** 2).sum(axis=3) if w is None else pad(np.asarray(w, dtype=np.float64)).sum(axis=3)
    return np.stack([s, q], axis=2).transpose(0, 3, 2, 1)


def ref_group_max(a, G):
    """torch.max over groups of G consecutive columns: (max, first index of it) [B, C, N / G]."""
    t = torch.from_numpy(np.ascontiguousarray(a)).reshape(a.shape[0], a.shape[1], -1, G)
    m, i = torch.max(t, dim=3)
    return m.numpy(), i.numpy().astype(np.int32)


def ref_knn(query, database, K):
    """[B, M, K] indices of the K nearest database points of each query by (d^2, index), by a lexsort."""
    q, d = np.asarray(query, dtype=np.int64), np.asarray(database, dtype=np.int64)
    out = np.empty((q.shape[0], q.shape[2], K), dtype=np.int32)
    for b in range(q.shape[0]):
        d2 = ((d[b][:, None, :] - q[b][:, :, None]) ** 2).sum(axis=0)            # [M, N]
        idx = np.broadcast_to(np.arange(d.shape[2]), d2.shape)
        for m in range(q.shape[2]):
            out[b, m] = np.lexsort((idx[m], d2[m]))[:K]
    return out


def ref_conv(x_nchw, W_okki, b, stride, pad):
    """float64 conv2d on the CPU: x [B, C, H, W], W [C_out, k, k, C_in] -> [B, C_out, Ho, Wo]."""
    x = torch.from_numpy(np.asarray(x_nchw, dtype=np.float64))
    w = torch.from_numpy(np.asarray(W_okki, dtype=np.float64)).permute(0, 3, 1, 2)
    bb = None if b is None else torch.from_numpy(np.asarray(b, dtype=np.float64))
    return torch.nn.functional.conv2d(x, w, bb, stride=stride, padding=pad).numpy()


def exact_bn_forward(s, q, M, gamma, beta, eps, momentum, rm, rv):
    """The exact values of chain_bn_kernel's forward for one channel from exact sums s, q over M points: mean, invstd,
    scale, shift, running mean, running var, each an mpmath number at 60 digits, and the absolute scale of shift."""
    with mpmath.workdps(60):
        f = lambda v: mpmath.mpf(Fraction(v).numerator) / Fraction(v).denominator
        mean = Fraction(int(s)) / M
        var = max(Fraction(int(q)) / M - mean * mean, Fraction(0))
        invstd = 1 / mpmath.sqrt(f(var + Fraction(float(np.float32(eps)))))
        scale = f(Fraction(float(gamma))) * invstd
        shift = f(Fraction(float(beta))) - f(mean) * scale
        mom = Fraction(float(np.float32(momentum)))     # eps and momentum reach the kernel as float32
        unbiased = var * M / (M - 1) if M > 1 else var
        run_mean = (1 - mom) * Fraction(float(rm)) + mom * mean
        run_var = (1 - mom) * Fraction(float(rv)) + mom * unbiased
        return dict(mean=f(mean), invstd=invstd, scale=scale, shift=shift, running_mean=f(run_mean),
                    running_var=f(run_var), shift_abs=abs(f(Fraction(float(beta)))) + abs(f(mean) * scale))


def exact_bn_backward(s, q, M, gamma, mean, invstd):
    """The exact dY coefficients k1, k2, k3 of chain_bn_kernel's backward for one channel (mean, invstd as stored in
    float32), and the absolute scale of k3."""
    g, mu, inv = (Fraction(float(v)) for v in (gamma, mean, invstd))
    k1 = g * inv
    k2 = -k1 * inv * Fraction(int(q)) / M
    k3 = -k1 * Fraction(int(s)) / M - k2 * mu
    return dict(k1=k1, k2=k2, k3=k3, k3_abs=abs(k1 * Fraction(int(s)) / M) + abs(k2 * mu))


def within_ulp(got, exact, abs_scale=0):
    """|got - exact| <= one float32 ulp of exact, or 2^-24 abs_scale where that is larger (a result that cancels);
    exact and abs_scale are Fractions or mpmath numbers."""
    with mpmath.workdps(60):
        mp = lambda v: mpmath.mpf(v.numerator) / v.denominator if isinstance(v, Fraction) else mpmath.mpf(v)
        e = mp(exact)
        tol = max(mpmath.mpf(float(np.spacing(np.float32(abs(float(e)))))), mp(abs_scale) * mpmath.mpf(2) ** -24)
        return abs(mpmath.mpf(float(got)) - e) <= tol


# ---------------------------------------------------------------------------------------------------------------------
# the dW split regimes the GPU tests cover: (B, N, C, K) -> which branch of dw_splits they hit

DW_CASES = [((1, 20, 64, 64), "single"),          # one 32-point chunk in all
            ((2, 77, 64, 64), "q_limited"),       # 6 chunks for 256 wanted splits
            ((8, 20480, 64, 64), "cap"),          # 1056 wanted, capped at 256
            ((2, 4133, 82, 736), "uneven"),       # 44 splits over 260 chunks
            ((3, 1000, 300, 40), "q_limited"),    # 212 wanted, 96 chunks; C off the 64 tile
            ((2, 4100, 1024, 1024), "uneven")]    # 5 splits over 258 chunks


def dw_regime(B, N, C, K):
    """Which branch of dw_splits decides (B, N, C, K): a single split, the chunk count Q, the 256 cap, or the CTA
    target with Q not a multiple of the splits."""
    tiles = -(-C // DW_TILE) * -(-K // DW_TILE)
    Q = B * -(-N // DW_PTS)
    want = -(-DW_TARGET_CTAS // tiles)
    s = dw_splits(B, N, C, K)
    if s == 1:
        return "single"
    if s == Q:
        return "q_limited"
    if want > DW_MAX_SPLITS:
        return "cap"
    return "uneven" if Q % s else "even"


def test_dw_split_cases_hit_every_branch():
    assert {dw_regime(*case) for case, _ in DW_CASES} == {"single", "q_limited", "cap", "uneven"}
    for case, want in DW_CASES:
        assert dw_regime(*case) == want, case
    assert dw_splits(1, 20, 64, 64) == 1 and dw_splits(2, 77, 64, 64) == 6 and dw_splits(8, 20480, 64, 64) == 256
    assert dw_splits(2, 4133, 82, 736) == 44 and 260 % 44 != 0


# ---------------------------------------------------------------------------------------------------------------------
# the generators and references on their own


@pytest.mark.parametrize("K, n_src", [(9, 2), (300, 4), (736, 2), (1024, 3), (65, 4), (7, 3)])
def test_split_rows_cover_the_rows_with_chunk_edges(K, n_src):
    w = split_rows(K, n_src)
    assert sum(w) == K and 1 <= len(w) <= n_src and all(c >= 1 for c in w)
    edges = np.cumsum(w)[:-1]
    if K > 64 and n_src >= 3:
        assert 64 in edges
    if n_src > 1 and K > 1:
        assert any(e % 64 for e in edges)


@pytest.mark.parametrize("C_out, C_in", [(1, 7), (82, 256), (256, 82), (2, 256), (1024, 1024)])
def test_sparse_weights_have_no_zero_row_or_column(C_out, C_in):
    W = sparse_weights(np.random.default_rng(C_out + C_in), C_out, C_in, 3, 2)
    assert np.all(np.any(W != 0, axis=0)) and np.all(np.any(W != 0, axis=1))
    assert_tf32(W)


# the shipped chains' widths (first, second, heads at 82 / 242 / 52 / 2 outputs) with a re-read activation each
CHAINS = [("first", 7, [32, 32, 32], [True, True, True], None),
          ("second", 64, [64, 64], [True, True], None),
          ("head_kitti", 736, [256, 256, 82], [True, True, False], 6),
          ("head_oxford", 736, [256, 256, 242], [True, True, False], 6),
          ("head_nuscenes", 736, [256, 256, 52], [True, True, False], 6),
          ("head_coarse", 736, [128, 128, 2], [True, True, False], 6)]


@pytest.mark.parametrize("spec", CHAINS, ids=[c[0] for c in CHAINS])
def test_chain_cases_are_exact_and_sensitive(spec):
    _, c_in, widths, relus, per_row = spec
    x, layers, out, pres = chain_case(np.random.default_rng(3), 2, 77, c_in, widths, relus, per_row=per_row)
    ref = torch.from_numpy(x).double()
    for W, b, relu in layers:
        ref = torch.einsum("ck,bkn->bcn", torch.from_numpy(W).double(), ref) + \
            torch.from_numpy(b).double()[None, :, None]
        ref = torch.relu(ref) if relu else ref
    assert np.array_equal(ref.numpy(), out)
    assert np.all(out == np.round(out)) and float(np.abs(out).max()) < EXACT


def test_reference_dw_and_partials_restate_the_sums():
    rng = np.random.default_rng(4)
    dy, x = ints(rng, (2, 5, 77), 3), ints(rng, (2, 6, 77), 3)
    dW, db = ref_dw(dy, x)
    want = sum(np.outer(dy[b, :, n], x[b, :, n]) for b in range(2) for n in range(77))
    assert np.array_equal(dW, want) and np.array_equal(db, dy.sum(axis=(0, 2)))
    p = ref_partials(dy)
    assert p.shape == (2, 2, 2, 5)
    assert np.array_equal(p[1, 1, 0], dy[1, :, 64:].sum(axis=1))
    assert np.array_equal(p[0, 0, 1], (dy[0, :, :64] ** 2).sum(axis=1))


def test_reference_knn_follows_distance_then_index():
    rng = np.random.default_rng(5)
    q = rng.integers(-2, 3, size=(2, 3, 9))
    d = rng.integers(-2, 3, size=(2, 3, 40))
    got = ref_knn(q, d, 17)
    for b in range(2):
        for m in range(9):
            key = [(int(((d[b, :, j] - q[b, :, m]) ** 2).sum()), j) for j in range(40)]
            assert [j for _, j in sorted(key)[:17]] == got[b, m].tolist()


def test_reference_group_max_takes_the_first_maximum():
    a = np.array([[[1, 3, 3, 0, 2, 2, 2, 2, -1]]], dtype=np.float32)
    m, i = ref_group_max(a, 3)
    assert m.tolist() == [[[3, 2, 2]]] and i.tolist() == [[[1, 1, 0]]]


def test_reference_conv_restates_the_definition():
    rng = np.random.default_rng(6)
    x, W = ints(rng, (1, 3, 5, 6), 2), ints(rng, (4, 3, 3, 3), 2)
    b = np.arange(4, dtype=np.float32)
    got = ref_conv(x, W, b, 2, 1)
    xp = np.pad(x, ((0, 0), (0, 0), (1, 1), (1, 1)))
    for o in range(4):
        for i in range(got.shape[2]):
            for j in range(got.shape[3]):
                want = (xp[0, :, 2 * i:2 * i + 3, 2 * j:2 * j + 3] * W[o].transpose(2, 0, 1)).sum() + b[o]
                assert got[0, o, i, j] == want


def test_exact_bn_matches_float64_where_float64_is_exact_enough():
    rng = np.random.default_rng(7)
    y = rng.integers(-20, 21, size=4096).astype(np.float64)
    s, q, M = y.sum(), (y * y).sum(), y.size
    e = exact_bn_forward(s, q, M, 1.5, -0.25, 1e-5, 0.1, 0.5, 2.0)
    var = y.var()
    assert abs(float(e["mean"]) - y.mean()) <= 1e-15
    assert abs(float(e["invstd"]) - 1 / np.sqrt(var + float(np.float32(1e-5)))) <= 1e-14
    assert abs(float(e["running_var"]) - (0.9 * 2.0 + float(np.float32(0.1)) * var * M / (M - 1))) <= 1e-6
    k = exact_bn_backward(s, q, M, 1.5, np.float32(0.25), np.float32(0.5))
    assert k["k1"] == Fraction(3, 4)
    assert within_ulp(np.float32(float(k["k2"])), k["k2"])
    assert within_ulp(np.float32(float(k["k3"])), k["k3"], k["k3_abs"])
    assert not within_ulp(np.nextafter(np.nextafter(np.float32(float(k["k2"])), np.float32(0)), np.float32(0)),
                          k["k2"])


def test_tf32_identity_holds_for_eleven_bits_and_fails_beyond():
    assert_tf32(np.arange(-2047, 2048, dtype=np.float32), np.float32([0.25, 3.5, 1023.5, 2 ** -20]))
    with pytest.raises(AssertionError):
        assert_tf32(np.float32([2049]))
    with pytest.raises(AssertionError):
        assert_sum_bound(np.array([2.0 ** 24]))


def test_one_dropped_chunk_passes_the_tolerance_gate_but_not_the_exact_comparison():
    """The motivation: at the `second` chain's test shape (B = 2, N = 4096, C = K = 64) a weight gradient that loses
    one 32-point chunk passes test_point_chain_gpu.py's gate |err| <= 16 2^-10 sum |terms| on every element, and
    fails the exact comparison outright."""
    rng = np.random.default_rng(8)
    dy, x = ints(rng, (2, 64, 4096), 2), ints(rng, (2, 64, 4096), 2)
    want, _ = ref_dw(dy, x)
    terms = np.einsum("bcn,bkn->ck", np.abs(dy).astype(np.float64), np.abs(x).astype(np.float64), optimize=True)
    assert_sum_bound(terms)
    lost = dy.copy()
    lost[1, :, 2048:2080] = 0                             # one 32-point chunk of sample 1 never summed
    got, _ = ref_dw(lost, x)
    bad = (np.abs(got - want) > 16 * 2.0 ** -10 * terms).mean()
    assert bad <= 1e-3                                    # the tolerance gate passes (in fact no element fails)
    assert bad == 0.0
    assert not np.array_equal(got, want)
    assert np.count_nonzero(got != want) > 0.9 * got.size
