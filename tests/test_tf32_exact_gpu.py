"""The fused TF32 kernels on exact integer cases (test_tf32_exact_cpu.py): every output and gradient equals the exact
reference bit for bit, whatever the kernel's tiling, split count or summation order, so a dropped, duplicated or
misplaced point, row or tap cannot hide under a TF32 tolerance.  Only BatchNorm's statistics, which divide and take
a square root, are compared within one float32 ulp of their exact values."""
import zlib
from fractions import Fraction

import numpy as np
import pytest
import torch

from deepi2p_b200 import _native, network, point_ops, resnet
from test_tf32_exact_cpu import (DW_CASES, PC_TILE, assert_no_zero_rows, assert_relu_live, assert_reread, assert_steps,
                                 assert_sum_bound, assert_tf32, chain_case, dw_splits, exact_bn_backward,
                                 exact_bn_forward, ints, mm, ref_conv, ref_dw, ref_group_max, ref_knn, ref_partials,
                                 sparse_weights, split_rows, within_ulp)

pytestmark = pytest.mark.gpu


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    return t.detach().cpu().numpy()


def assert_exact(got, want, what):
    g = host(got).astype(np.float64) if isinstance(got, torch.Tensor) else np.asarray(got, dtype=np.float64)
    want = np.asarray(want, dtype=np.float64)
    assert g.shape == want.shape, f"{what}: shape {g.shape}, want {want.shape}"
    bad = g != want
    assert not bad.any(), f"{what}: {int(bad.sum())} of {bad.size} elements differ, the first at " \
                          f"{tuple(int(i) for i in np.argwhere(bad)[0])}: {g[bad][0]!r} != {want[bad][0]!r}"


def dropout(rng, layer, B, C, N):
    """(drop_state, p = 0.5) and the kernel's keep mask: the kept values are scaled by exactly 2."""
    state = point_ops.new_dropout_state(int(rng.integers(1, 2 ** 40)), torch.device("cuda"))
    return (state, 0.5), host(point_ops.point_chain_dropout_mask(state, layer, 0.5, B, C, N)).astype(np.float64)


def act_stats(rng, C, amp_shift=2):
    """A BN layer's [4, C] statistics written by the test: integer mean, power-of-two invstd, scale 1 or 2, integer
    shift (the act transform reads scale and shift; the act-grad epilogue also mean and invstd)."""
    st = np.stack([rng.integers(-2, 3, C), 2.0 ** -rng.integers(0, 3, C), rng.choice([1.0, 2.0], C),
                   rng.integers(-1, amp_shift + 1, C)]).astype(np.float32)
    assert_tf32(st)
    return st


class Operand:
    """An operand of the chain kernels in one of the transforms and its exact value x [B, K, N]; step is the finest
    power of two its values are multiples of."""

    def __init__(self, rng, mode, B, N, K, n_src=1, group=None, amp=2, layer=0):
        self.keep, self.step, self.widths = [], 1.0, [K]
        if mode == "plain":
            self.widths = split_rows(K, n_src)
            srcs = [ints(rng, (B, w, N), amp) for w in self.widths]
            self.keep = [cu(s) for s in srcs]
            self.table, self.n_src = point_ops._chain_operand(self.keep), len(srcs)
            self.x = np.concatenate(srcs, axis=1).astype(np.float64)
        elif mode in ("act", "act_drop"):
            y = ints(rng, (B, K, N), amp + 1)
            st = act_stats(rng, K)
            z = st[2][None, :, None] * y.astype(np.float64) + st[3][None, :, None]
            assert_relu_live(z, (0, 2))
            self.x = np.maximum(z, 0.0)
            drop = None
            if mode == "act_drop":
                drop, mask = dropout(rng, layer, B, K, N)
                self.x = self.x * 2.0 * mask
            self.keep = [cu(y), cu(st)] + ([drop[0]] if drop else [])
            self.table = point_ops._chain_operand([self.keep[0]], point_ops._OP_ACT, self.keep[1], drop=drop,
                                                  layer=layer)
            self.n_src = 1
        elif mode == "bn_grad":
            dz, y = ints(rng, (B, K, N), amp), ints(rng, (B, K, N), amp)
            k = np.stack([rng.choice([1.0, 2.0, -1.0], K), rng.choice([0.5, -0.5, 1.0], K),
                          rng.choice([0.25, -0.75, 0.0], K)]).astype(np.float32)
            self.x = k[0][None, :, None] * dz + k[1][None, :, None] * y.astype(np.float64) + k[2][None, :, None]
            self.step = 0.25
            self.keep = [cu(dz), cu(y), cu(k)]
            self.table = point_ops._chain_operand([self.keep[0]], point_ops._OP_BN_GRAD, self.keep[2], self.keep[1])
            self.n_src = 1
        elif mode == "max_grad":
            t = cu(rng.integers(0, 3, (B, K, N)).astype(np.float32))     # small integers: ties in most groups
            _, mx, idx = point_ops._chain_group_max(point_ops._chain_operand([t]), B, N, K, group, False)
            rm, ri = ref_group_max(host(t), group)
            assert_exact(mx, rm, "group max")
            assert_exact(idx, ri, "group max index")
            g = ints(rng, (B, K, N // group), amp)
            self.x = np.zeros((B, K, N))
            b, c, j = np.meshgrid(np.arange(B), np.arange(K), np.arange(N // group), indexing="ij")
            self.x[b, c, j * group + ri] = g
            self.keep = [t, cu(g), idx]
            self.table, self.n_src = point_ops._chain_max_grad_operand(self.keep[1], idx, group), 1
        else:
            raise ValueError(mode)
        assert_tf32(self.x)
        assert_steps(self.x, self.step)
        assert_no_zero_rows(self.x if mode != "max_grad" else self.x.reshape(B, K, -1, group).any(3), (0, 2),
                            "operand row")


# ---------------------------------------------------------------------------------------------------------------------
# 1. point_chain primitives

# (B, N, K, C, n_src, operand mode, epilogue, bias, add_group (0: none), weights (False: elementwise))
GEMM_CASES = [
    (1, 1, 1, 1, 1, "plain", "write", True, 0, True),
    (2, 63, 7, 15, 3, "plain", "stats", False, 1, True),
    (1, 64, 8, 16, 2, "act", "write", True, 0, True),
    (2, 65, 9, 17, 2, "plain", "act_grad", False, 0, True),
    (8, 77, 63, 82, 1, "act_drop", "stats", True, 1, True),
    (2, 4133, 64, 256, 1, "bn_grad", "write", False, 0, True),
    (1, 65, 65, 256, 4, "plain", "stats", True, 0, True),
    (2, 77, 300, 82, 4, "plain", "act_grad", True, 1, True),
    (1, 4133, 736, 64, 1, "act", "stats", False, 0, True),
    (2, 65, 1024, 17, 3, "plain", "write", True, 0, True),
    (2, 77, 16, 16, 1, "max_grad", "act_grad", False, 0, True),
    (8, 20480, 64, 64, 1, "act_drop", "stats", True, 0, True),
    # wider than 256 rows: row blocks over grid z, and a grouped additive term
    (2, 77, 64, 257, 2, "plain", "stats", True, 7, True),
    (1, 65, 300, 300, 1, "act_drop", "write", True, 1, True),
    (2, 130, 82, 512, 1, "bn_grad", "stats", False, 13, True),
    (1, 64, 9, 1024, 2, "plain", "act_grad", True, 0, True),
    (2, 20480, 32, 64, 1, "plain", "write", False, 16, True),
    # elementwise (no weights): the transformed operand itself
    (2, 77, 17, 17, 1, "act_drop", "write", False, 0, False),
    (1, 65, 82, 82, 1, "bn_grad", "stats", True, 1, False),
    (2, 77, 16, 16, 1, "max_grad", "act_grad", False, 0, False),
]


def _gemm_id(c):
    B, N, K, C, n, mode, ep, bias, ag, w = c
    return f"B{B}_N{N}_K{K}_C{C}_{n}src_{mode}_{ep}" + ("_bias" if bias else "") + (f"_add{ag}" if ag else "") + \
        ("" if w else "_elementwise")


@pytest.mark.parametrize("case", GEMM_CASES, ids=[_gemm_id(c) for c in GEMM_CASES])
def test_chain_gemm_exact(case):
    B, N, K, C, n_src, mode, ep, with_bias, add_group, with_w = case
    rng = np.random.default_rng(zlib.crc32(_gemm_id(case).encode()))
    op = Operand(rng, mode, B, N, K, n_src, group=7 if mode == "max_grad" else None)
    W = sparse_weights(rng, C, K, 8, 2 if K <= 300 else 1) if with_w else None
    bias = rng.integers(-3, 4, C).astype(np.float32) if with_bias else None
    add = ints(rng, (B, C, N // add_group), 3) if add_group else None
    v = mm(W, op.x) if with_w else op.x.copy()
    terms = (mm(np.abs(W), np.abs(op.x)) if with_w else np.abs(op.x))
    if bias is not None:
        v, terms = v + bias[None, :, None], terms + np.abs(bias)[None, :, None]
    if add is not None:
        a = np.repeat(add, add_group, axis=2)
        v, terms = v + a, terms + np.abs(a)
    assert_sum_bound(terms, op.step, aim=False)
    epi = {"write": point_ops._EP_WRITE, "stats": point_ops._EP_STATS, "act_grad": point_ops._EP_ACT_GRAD}[ep]
    act = act_y = None
    w = None
    if ep == "act_grad":                           # the gradient v of a BN layer's output, through its ReLU / dropout
        st = act_stats(rng, C, amp_shift=3)
        ey = ints(rng, (B, C, N), 3)
        keep = st[2][None, :, None] * ey.astype(np.float64) + st[3][None, :, None] > 0
        assert_relu_live(np.where(keep, 1.0, -1.0), (0, 2))
        drop = None
        if C % 2 == 0:
            drop, mask = dropout(rng, 2, B, C, N)
            keep = keep & (mask > 0)
        v = np.where(keep, v * (2.0 if drop else 1.0), 0.0)
        w = v * ((ey - st[0][None, :, None]) * st[1][None, :, None])
        assert float(np.abs(w).max()) / (op.step * 0.25) < 2.0 ** 24
        st_t, act_y = cu(st), cu(ey)
        op.keep += [st_t, act_y]
        act = point_ops._chain_act_row(st_t, drop, 2)
    packed = point_ops._chain_pack(cu(W), op.widths) if with_w else None
    keep = [cu(bias) if bias is not None else None, cu(add) if add is not None else None]
    out, part = point_ops._chain_gemm(op.table, op.n_src, packed, keep[0], keep[1], C, B, N, epi, act, act_y,
                                      add_group=max(add_group, 1))
    T = -(-N // PC_TILE)
    part = part[:B * T * 2 * C * 8].view(torch.float64).reshape(B, T, 2, C).clone() if part is not None else None
    torch.cuda.synchronize()
    assert_exact(out, v, "out")
    if ep != "write":
        assert_exact(part, ref_partials(v, w), "per-tile partial sums")


# (B, N, C, K), dY's transform, X's transform, X's sources
DW_RUNS = [(c, "plain", "plain", 1) for c, _ in DW_CASES] + [
    ((2, 4133, 82, 736), "bn_grad", "act_drop", 1),
    ((3, 1000, 300, 40), "plain", "plain", 4),
    ((2, 77, 64, 64), "bn_grad", "act", 1),
    ((1, 20, 64, 64), "plain", "act_drop", 1),
    ((2, 130, 17, 9), "max_grad", "plain", 3),
]


@pytest.mark.parametrize("run", DW_RUNS, ids=[f"B{r[0][0]}_N{r[0][1]}_C{r[0][2]}_K{r[0][3]}_{r[1]}_{r[2]}_{r[3]}src"
                                              for r in DW_RUNS])
def test_chain_dw_exact(run):
    (B, N, C, K), dy_mode, x_mode, n_src = run
    S = dw_splits(B, N, C, K)
    lib = _native.load()
    assert lib.point_chain_dw_workspace_bytes(B, N, C, K) == S * C * K * 4 + S * C * 8 + 16
    rng = np.random.default_rng(B * N + C * K)
    amp = 1 if B * N > 10000 else 2
    dy = Operand(rng, dy_mode, B, N, C, group=13 if dy_mode == "max_grad" else None, amp=amp)
    x = Operand(rng, x_mode, B, N, K, n_src, amp=amp, layer=1)
    want, want_db = ref_dw(dy.x, x.x)
    assert_sum_bound(ref_dw(np.abs(dy.x), np.abs(x.x))[0], dy.step * x.step, aim=False)
    dW, db = point_ops._chain_dw(dy.table, x.table, x.n_src, B, N, C, K, True)
    assert_exact(dW, want, f"dW ({S} splits)")
    assert_exact(db, want_db, "db")


# (B, N, C): G = B * ceil(N / 64) tiles below and above the kernel's 256 threads; M = B N a power of two or not
BN_CASES = [(2, 4133, 82), (8, 20480, 17), (4, 4096, 300), (1, 64, 1024), (3, 77, 5)]


def _bn_module(rng, C, eps=1e-5):
    norm = torch.nn.BatchNorm1d(C, eps=eps, momentum=0.1).cuda()
    with torch.no_grad():
        norm.weight.copy_(cu(rng.choice([0.5, 1.0, 1.5, 2.0], C).astype(np.float32)))
        norm.bias.copy_(cu(rng.choice([-0.25, 0.0, 0.5, 3.0], C).astype(np.float32)))
        norm.running_mean.copy_(cu(rng.normal(0, 1, C).astype(np.float32)))
        norm.running_var.copy_(cu(rng.uniform(0.5, 2, C).astype(np.float32)))
    return norm


@pytest.mark.parametrize("B, N, C", BN_CASES, ids=[f"B{b}_N{n}_C{c}" for b, n, c in BN_CASES])
def test_chain_bn_forward_within_one_ulp(B, N, C):
    rng = np.random.default_rng(B + N + C)
    T = -(-N // PC_TILE)
    y = ints(rng, (B, C, N), 6) + rng.integers(-4, 5, C).astype(np.float32)[None, :, None]
    part = ref_partials(y)
    norm = _bn_module(rng, C)
    rm, rv = host(norm.running_mean), host(norm.running_var)
    nbt = int(norm.num_batches_tracked)
    stats = torch.empty((4, C), dtype=torch.float32, device="cuda")
    point_ops._chain_bn(cu(part), B, N, C, norm, stats, grad=False)
    st, grm, grv = host(stats), host(norm.running_mean), host(norm.running_var)
    s, q, M = part[:, :, 0].sum(axis=(0, 1)), part[:, :, 1].sum(axis=(0, 1)), B * N
    assert B * T == part.shape[0] * part.shape[1]
    gamma, beta = host(norm.weight), host(norm.bias)
    for c in range(C):
        e = exact_bn_forward(s[c], q[c], M, gamma[c], beta[c], norm.eps, norm.momentum, rm[c], rv[c])
        for name, got, scale in (("mean", st[0, c], 0), ("invstd", st[1, c], 0), ("scale", st[2, c], 0),
                                 ("shift", st[3, c], e["shift_abs"]), ("running_mean", grm[c], 0),
                                 ("running_var", grv[c], 0)):
            assert within_ulp(got, e[name], scale), f"{name}[{c}] = {got!r}, exact {e[name]}"
        if M & (M - 1) == 0:                       # M a power of two: the mean is representable and must be exact
            assert Fraction(float(st[0, c])) == Fraction(int(s[c]), M)
    assert int(norm.num_batches_tracked) == nbt + 1


@pytest.mark.parametrize("B, N, C", BN_CASES, ids=[f"B{b}_N{n}_C{c}" for b, n, c in BN_CASES])
def test_chain_bn_backward_exact_and_within_one_ulp(B, N, C):
    rng = np.random.default_rng(B * N + C)
    T = -(-N // PC_TILE)
    part = np.stack([rng.integers(-3000, 3001, (B, T, C)), rng.integers(-3000, 3001, (B, T, C))], axis=2)
    part = part.astype(np.float64)
    norm = _bn_module(rng, C)
    st = act_stats(rng, C)
    st[1] = 2.0 ** -rng.integers(0, 4, C)
    dgamma, dbeta, coef = point_ops._chain_bn(cu(part), B, N, C, norm, cu(st), grad=True)
    s, q = part[:, :, 0].sum(axis=(0, 1)), part[:, :, 1].sum(axis=(0, 1))
    assert np.abs(s).max() < 2 ** 24 and np.abs(q).max() < 2 ** 24
    assert_exact(dbeta, s, "dbeta")
    assert_exact(dgamma, q, "dgamma")
    k, gamma = host(coef), host(norm.weight)
    for c in range(C):
        e = exact_bn_backward(s[c], q[c], B * N, gamma[c], st[0, c], st[1, c])
        assert Fraction(float(k[0, c])) == e["k1"], f"k1[{c}]"
        assert within_ulp(k[1, c], e["k2"]), f"k2[{c}] = {k[1, c]!r}, exact {float(e['k2'])}"
        assert within_ulp(k[2, c], e["k3"], e["k3_abs"]), f"k3[{c}] = {k[2, c]!r}, exact {float(e['k3'])}"


# (B, N, C, G, operand mode)
GROUP_CASES = [(2, 77, 17, 7, "act_drop"), (1, 20480, 64, 16, "bn_grad"), (8, 4096, 5, 4096, "plain"),
               (2, 65, 3, 1, "act"), (2, 130, 300, 13, "plain")]


@pytest.mark.parametrize("B, N, C, G, mode", GROUP_CASES, ids=[f"B{c[0]}_N{c[1]}_C{c[2]}_G{c[3]}_{c[4]}"
                                                             for c in GROUP_CASES])
def test_chain_group_max_and_sum_exact(B, N, C, G, mode):
    rng = np.random.default_rng(N + G)
    op = Operand(rng, mode, B, N, C, amp=1)
    act, mx, idx = point_ops._chain_group_max(op.table, B, N, C, G, True)
    rm, ri = ref_group_max(op.x.astype(np.float32), G)
    assert_exact(act, op.x, "act")
    assert_exact(mx, rm, "group max")
    assert_exact(idx, ri, "group max index")
    assert_exact(point_ops._chain_group_sum(op.table, B, N, C, G), op.x.reshape(B, C, -1, G).sum(axis=3),
                 "group sum")


# ---------------------------------------------------------------------------------------------------------------------
# 2. autograd paths, exact end to end


def _linear_layer(rng, c_in, C, amp=1):
    layer = network._PointLayer(c_in, C, False).cuda()
    W = sparse_weights(rng, C, c_in, 6, amp)
    b = rng.integers(-3, 4, C).astype(np.float32)
    with torch.no_grad():
        layer.conv.weight.copy_(cu(W[:, :, None]))
        layer.conv.bias.copy_(cu(b))
    return layer, W, b


# (B, N, source widths, cols (None: in order), c_in, C, add_group (0: no add), entry point)
BRANCH_CASES = [
    (2, 77, (64, 100, 36, 100), None, 300, 82, 0, "branch"),
    (1, 4133, (32, 64), None, 736, 256, 1, "chain"),                 # in_col = 640, the head's sources
    (2, 65, (5, 9, 3), (12, 0, 9), 17, 17, 0, "branch"),
    (2, 77, (40, 24), (24, 0), 100, 300, 11, "branch"),
    (8, 20480, (32, 32), None, 64, 64, 0, "branch"),
]


@pytest.mark.parametrize("case", BRANCH_CASES, ids=["4_sources", "in_col", "cols_out_of_order", "add_group_11",
                                                    "shipped_B8_N20480"])
def test_linear_point_branch_exact_end_to_end(case):
    B, N, widths, cols, c_in, C, add_group, entry = case
    rng = np.random.default_rng(sum(widths) + N)
    layer, W, b = _linear_layer(rng, c_in, C)
    if cols is None:
        cols = [c_in - sum(widths) + sum(widths[:i]) for i in range(len(widths))]
    xs = [ints(rng, (B, w, N), 2) for w in widths]
    srcs = [cu(x).requires_grad_() for x in xs]
    add = ints(rng, (B, C, N // add_group), 3) if (add_group or sum(widths) < c_in) else None
    G = max(add_group, 1)
    add_t = cu(add).requires_grad_() if add is not None else None
    if entry == "chain":
        out = point_ops.point_chain(srcs, [layer], True, add=add_t, in_col=cols[0])
    else:
        out = point_ops.point_branch(srcs, [layer], cols=list(cols), add=add_t, add_group=G)
    g = ints(rng, (B, C, N), 2)
    out.backward(cu(g))
    Wu = np.concatenate([W[:, c:c + w] for c, w in zip(cols, widths)], axis=1)
    x = np.concatenate(xs, axis=1).astype(np.float64)
    want = mm(Wu, x) + b[None, :, None] + (np.repeat(add, G, axis=2) if add is not None else 0)
    assert_sum_bound(mm(np.abs(Wu), np.abs(x)) + 3 + (3 if add is not None else 0), aim=False)
    assert_exact(out, want, "out")
    dWu, db = ref_dw(g, x)
    dW = np.zeros((C, c_in))
    r = 0
    for c, w in zip(cols, widths):
        dW[:, c:c + w] = dWu[:, r:r + w]
        r += w
    assert_exact(layer.conv.weight.grad[:, :, 0], dW, "dW")
    assert_exact(layer.conv.bias.grad, db, "db")
    gx = mm(Wu.T, g)
    r = 0
    for i, (s, w) in enumerate(zip(srcs, widths)):
        assert_exact(s.grad, gx[:, r:r + w], f"source {i} gradient")
        r += w
    if add is not None:
        assert_exact(add_t.grad, g.reshape(B, C, -1, G).sum(axis=3), "add gradient")


def test_max_group_branch_exact_with_dyadic_batch_statistics():
    """A BN layer whose batch statistics are dyadic: eps = 0, and each channel's pre-norm values are m +- d and
    m +- 3d in the proportions 5 : 3 over M = 256 points, so mean and var are exact, var = 4 d^2 and invstd =
    1 / (2 d).  The activations, the group max and its index (the kernel's, checked through dgamma / dbeta against
    torch.max's rule), the running mean and dgamma / dbeta are then exact."""
    rng = np.random.default_rng(11)
    B, N, C, G, d = 2, 128, 16, 16, 2.0
    M = B * N
    perm, sign = rng.permutation(C), rng.choice([-1.0, 1.0], C)
    layer = network._PointLayer(C, C, True).cuda()
    layer.norm.eps = 0.0
    W = np.zeros((C, C), dtype=np.float32)
    W[np.arange(C), perm] = sign
    b = rng.integers(-3, 4, C).astype(np.float32)
    gamma, beta = rng.choice([1.0, 2.0, 3.0], C).astype(np.float32), rng.integers(-1, 3, C).astype(np.float32)
    with torch.no_grad():
        layer.conv.weight.copy_(cu(W[:, :, None]))
        layer.conv.bias.copy_(cu(b))
        layer.norm.weight.copy_(cu(gamma))
        layer.norm.bias.copy_(cu(beta))
    base = np.array([1.0] * (5 * M // 16) + [-1.0] * (5 * M // 16) + [3.0] * (3 * M // 16) + [-3.0] * (3 * M // 16))
    x = np.stack([rng.permutation(base).reshape(B, N) * d + rng.integers(-4, 5) for _ in range(C)], axis=1)
    x = x.astype(np.float32)
    src = cu(x).requires_grad_()
    act, mx = point_ops.point_branch([src], [layer], max_group=G, output="both")
    y = mm(W, x) + b[None, :, None]
    mean, invstd = y.mean(axis=(0, 2)), 1.0 / (2 * d)
    assert np.all(y.var(axis=(0, 2)) == 4 * d * d)
    a = np.maximum((y - mean[None, :, None]) * invstd * gamma[None, :, None] + beta[None, :, None], 0.0)
    assert_relu_live(a, (0, 2))
    rm, ri = ref_group_max(a.astype(np.float32), G)
    assert_exact(act, a, "activations")
    assert_exact(mx, rm, "group max")
    for c in range(C):                           # from a zero running mean
        assert within_ulp(host(layer.norm.running_mean)[c], Fraction(float(np.float32(0.1))) * Fraction(mean[c]))
    gm = ints(rng, (B, C, N // G), 2)
    mx.backward(cu(gm))
    dz = np.zeros((B, C, N))
    bb, cc, jj = np.meshgrid(np.arange(B), np.arange(C), np.arange(N // G), indexing="ij")
    dz[bb, cc, jj * G + ri] = gm
    dz = np.where(a > 0, dz, 0.0)
    xhat = (y - mean[None, :, None]) * invstd
    assert_exact(layer.norm.bias.grad, dz.sum(axis=(0, 2)), "dbeta")
    assert_exact(layer.norm.weight.grad, (dz * xhat).sum(axis=(0, 2)), "dgamma")


CP_CASES = [(256, 128, 128), (256, 512, 128), (300, 40, 77), (1024, 1024, 33)]


@pytest.mark.parametrize("C, K, M", CP_CASES, ids=[f"C{c}_K{k}_M{m}" for c, k, m in CP_CASES])
def test_channel_product_exact(C, K, M):
    rng = np.random.default_rng(C + K + M)
    B = 2
    W, x, g = ints(rng, (C, K), 1), ints(rng, (B, K, M), 2), ints(rng, (B, C, M), 2)
    Wt, xt = cu(W).requires_grad_(), cu(x).requires_grad_()
    out = point_ops.channel_product(Wt, xt)
    out.backward(cu(g))
    assert_exact(out, mm(W, x), "out")
    assert_exact(Wt.grad, ref_dw(g, x)[0], "dW")
    assert_exact(xt.grad, mm(W.T, g), "dx")


# ---------------------------------------------------------------------------------------------------------------------
# 3. inference ops

MLP_CASES = [("first", 7, [32, 32, 32], [True, True, True], None, 2, 4133),
             ("second", 64, [64, 64], [True, True], None, 8, 20480),
             ("head_kitti", 736, [256, 256, 82], [True, True, False], 6, 2, 65),
             ("head_oxford", 736, [256, 256, 242], [True, True, False], 6, 1, 63),
             ("head_nuscenes", 736, [256, 256, 52], [True, True, False], 6, 2, 4133),
             ("head_coarse", 736, [128, 128, 2], [True, True, False], 6, 2, 1),
             ("k_tail", 65, [17, 9], [True, False], None, 2, 77)]


@pytest.mark.parametrize("case", MLP_CASES, ids=[c[0] for c in MLP_CASES])
def test_pointwise_mlp_exact(case):
    name, c_in, widths, relus, per_row, B, N = case
    rng = np.random.default_rng(c_in + N)
    x, layers, want, _ = chain_case(rng, B, N, c_in, widths, relus, per_row=per_row)
    srcs = [cu(s) for s in np.split(x, np.cumsum(split_rows(c_in, 3))[:-1], axis=1)]
    lt = [(cu(W), cu(b), r) for W, b, r in layers]
    with torch.no_grad():
        assert_exact(point_ops.pointwise_mlp(srcs, lt), want, "activations")
        c_split = min(2, widths[-1])
        pa, pb, sc = point_ops.pointwise_mlp(srcs, lt, output="argmax", c_split=c_split, return_scores=True)
    assert_exact(sc, want, "scores")
    assert_exact(pa, np.argmax(want[:, :c_split], axis=1), "arg-max below c_split (first maximal index)")
    if widths[-1] > c_split:
        assert_exact(pb, np.argmax(want[:, c_split:], axis=1), "arg-max from c_split (first maximal index)")


@pytest.mark.parametrize("N", [1, 65, 20480])
def test_pointwise_mlp_max_exact(N):
    rng = np.random.default_rng(N)
    B = 2 if N > 1000 else 3
    x, layers, want, _ = chain_case(rng, B, N, 15, [64, 128, 40], [True, True, False])
    with torch.no_grad():
        got = point_ops.pointwise_mlp_max([cu(x[:, :3]), cu(x[:, 3:])], [(cu(W), cu(b), r) for W, b, r in layers])
    assert_exact(got, want.max(axis=2, keepdims=True), "max over the columns")


@pytest.mark.parametrize("K", [1, 3, 16, 17, 32])
def test_knn_fusion_exact(K):
    rng = np.random.default_rng(K)
    B, M, Nd, C = 2, 45, 70, 6
    q = rng.integers(-3, 4, (B, 3, M)).astype(np.float32)        # integer coordinates: distances tie
    d = rng.integers(-3, 4, (B, 3, Nd)).astype(np.float32)
    f = ints(rng, (B, C, Nd), 2)
    idx = ref_knn(q, d, K)
    grouped = np.concatenate([d[np.arange(B)[:, None, None], :, idx].transpose(0, 3, 1, 2) - q[:, :, :, None],
                              f[np.arange(B)[:, None, None], :, idx].transpose(0, 3, 1, 2)], axis=1)   # [B,3+C,M,K]
    flat = grouped.reshape(B, 3 + C, M * K)
    _, before, h, _ = chain_case(rng, B, M * K, 3 + C, [24, 12], [True, True], x=flat)
    assert_reread(h)
    hm = h.reshape(B, 12, M, K).max(axis=3)
    cat = np.concatenate([np.repeat(hm, K, axis=2), h], axis=1)                  # [max; x], per (m, k) column
    _, after, out, _ = chain_case(rng, B, M * K, 24, [20, 8], [True, False], per_row=3, x=cat)
    want = out.reshape(B, 8, M, K).max(axis=3)
    with torch.no_grad():
        out, gidx = point_ops.knn_fusion(cu(q), cu(d), cu(f), K, ([(cu(W), cu(b), r) for W, b, r in before],
                                                                  [(cu(W), cu(b), r) for W, b, r in after]),
                                         return_idx=True)
    assert_exact(gidx, idx, "kNN indices (d^2, then index)")
    assert_exact(out, want, "kNN fusion output")


NODE_CASES = [(2, 77, [600, 40], "two_passes"), (9, 65, [64, 17], "B9"), (4, 33, [1024, 8], "width_1024")]


@pytest.mark.parametrize("B, M, widths, name", NODE_CASES, ids=[c[3] for c in NODE_CASES])
def test_node_mlp_exact(B, M, widths, name):
    rng = np.random.default_rng(B * M)
    dense, ps = ints(rng, (B, 20, M), 2), ints(rng, (B, 300, 1), 2)    # a per-sample source, applied by fma chain
    x = np.concatenate([dense[:, :12], np.broadcast_to(ps, (B, 300, M)), dense[:, 12:]], axis=1)
    _, layers, want, _ = chain_case(rng, B, M, 320, widths, [True, False], per_row=4, x=x)
    with torch.no_grad():
        got = point_ops.node_mlp([cu(dense[:, :12]), cu(ps[:, :, 0]), cu(dense[:, 12:])],
                                 [(cu(W), cu(b), r) for W, b, r in layers])
    assert_exact(got, want, "node_mlp")


# (name, B, H, W, C_in, C_out, k, stride, extra): extra in None, "residual", "shortcut", "stage_end", "last", "stem"
CONV_CASES = [("plain_odd_stride2", 2, 9, 11, 64, 40, 3, 2, None),
              ("residual", 1, 7, 5, 32, 64, 3, 1, "residual"),
              ("shortcut", 2, 5, 7, 64, 128, 3, 1, "shortcut"),
              ("stage_end", 1, 3, 3, 32, 256, 3, 1, "stage_end"),
              ("last_1x1_output", 2, 1, 1, 64, 72, 3, 1, "last"),
              ("m_127", 1, 1, 127, 32, 64, 3, 1, None),
              ("m_129", 1, 3, 43, 32, 24, 1, 1, None),
              ("stem", 2, 19, 23, 3, 64, 7, 2, "stem")]


@pytest.mark.parametrize("case", CONV_CASES, ids=[c[0] for c in CONV_CASES])
def test_conv2d_fused_exact(case):
    name, B, H, Wd, C_in, C_out, k, stride, extra = case
    rng = np.random.default_rng(len(name) * 100 + H)
    x = ints(rng, (B, C_in, H, Wd), 2)
    W = ints(rng, (C_out, k, k, C_in), 1)
    b = rng.integers(-8, 9, C_out).astype(np.float32)
    want = ref_conv(x, W, b, stride, k // 2)
    assert_no_zero_rows(W, (0, 3), "conv tap")
    assert_sum_bound(ref_conv(np.abs(x), np.abs(W), np.abs(b), stride, k // 2), aim=False)
    kw = {}
    short = None
    if extra == "residual":
        res = ints(rng, (B, C_out) + want.shape[2:], 3)
        want = want + res
        kw["residual"] = cu(res.transpose(0, 2, 3, 1))
    if extra == "shortcut":
        xs = ints(rng, (B, 32, 2 * want.shape[2] - 1, 2 * want.shape[3]), 2)
        Wsc = ints(rng, (C_out, 1, 1, 32), 1)
        bsc = rng.integers(-2, 3, C_out).astype(np.float32)
        want = want + ref_conv(xs, Wsc, bsc, 2, 0)
        short = (cu(Wsc), cu(bsc))
        kw.update(shortcut=cu(xs.transpose(0, 2, 3, 1)), shortcut_stride=2)
    relu = extra != "last"
    want = np.maximum(want, 0) if relu else want
    layer = resnet.pack_conv(cu(W), cu(b), shortcut=short)
    xin = cu(x) if extra == "stem" else cu(x.transpose(0, 2, 3, 1))
    with torch.no_grad():
        if extra == "stage_end":
            out, cm = resnet.conv2d_fused(xin, layer, stride, channel_major=True, **kw)
            assert_exact(cm, want.reshape(B, C_out, -1), "channel-major output")
        elif extra == "last":
            _, cm = resnet.conv2d_fused(xin, layer, stride, relu=False, channel_major=True, nhwc=False, **kw)
            out = cm.reshape(B, C_out, *want.shape[2:]).permute(0, 2, 3, 1)
        else:
            out = resnet.conv2d_fused(xin, layer, stride, nchw_input=extra == "stem", **kw)
    assert_exact(out, want.transpose(0, 2, 3, 1), "NHWC output")


@pytest.mark.parametrize("B, H, W, C", [(2, 9, 11, 64), (1, 1, 1, 8), (3, 16, 7, 32)])
def test_max_pool_and_channel_mean_exact(B, H, W, C):
    rng = np.random.default_rng(H * W)
    x = rng.integers(-3, 4, (B, H, W, C)).astype(np.float32)         # small integers: ties in most windows
    want = torch.nn.functional.max_pool2d(torch.from_numpy(x).double().permute(0, 3, 1, 2), 3, 2, 1)
    assert_exact(resnet.max_pool_3x3s2(cu(x)), want.permute(0, 2, 3, 1).numpy(), "max pool")
    y = ints(rng, (B, C, H * W * 37), 100)
    s = y.astype(np.int64).sum(axis=2)
    assert_exact(resnet.channel_mean(cu(y)), np.float32(s / y.shape[2]), "channel mean")
