"""The packed weight format of the fused TF32 ops (DESIGN.md 4.21): every float that pack_pointwise_mlp,
pack_knn_fusion, pack_pointwise_mlp_max and pack_node_mlp write, bit for bit against a numpy restatement of the
layout: the m16n8k8 A-fragment order of tf32_mma.cuh's a_frag_row_col, oracle_pointwise.tf32_round, rows padded to 16
and k tiles to 8 with zeros, the transposed blocks and the padded biases."""
import numpy as np
import pytest
import torch

from deepi2p_b200 import point_ops
from oracle_pointwise import tf32_round

pytestmark = pytest.mark.gpu


def pad(x, m):
    return (x + m - 1) // m * m


def a_frag(W, KT):
    """W [R][K] -> its A-fragment order [m tile][k tile][lane][4] over pad16(R) rows and KT k tiles, rounded to TF32,
    zero in the padding."""
    R = pad(W.shape[0], 16)
    Wp = np.zeros((R, KT * 8), dtype=np.float32)
    Wp[:W.shape[0], :W.shape[1]] = tf32_round(W)
    e = np.arange(R * KT * 8)
    i, lane, tile = e & 3, (e >> 2) & 31, e >> 7
    row = (tile // KT) * 16 + (lane >> 2) + (i & 1) * 8
    col = (tile % KT) * 8 + (lane & 3) + (i >> 1) * 4
    return Wp[row, col]


def transposed(W, Cpad):
    """W [C][K] -> [K][Cpad], rounded to TF32, zero in the padding."""
    out = np.zeros((W.shape[1], Cpad), dtype=np.float32)
    out[:, :W.shape[0]] = tf32_round(W).T
    return out.ravel()


def bias(b, C):
    out = np.zeros(pad(C, 16), dtype=np.float32)
    if b is not None:
        out[:C] = b
    return out


def chain(layers, k0_pad):
    """Each layer's weights then its bias: layer 0 over k0_pad input rows, each later layer over its predecessor's
    padded width (the columns past its width are zero)."""
    parts, kt = [], k0_pad // 8
    for W, b, _ in layers:
        parts += [a_frag(W, kt), bias(b, W.shape[0])]
        kt = pad(W.shape[0], 16) // 8
    return parts


def random_layers(rng, c_in, widths, no_bias=()):
    layers = []
    for i, c in enumerate(widths):
        W = rng.normal(0, 1, (c, c_in)).astype(np.float32)
        W.ravel()[::7] = np.float32(1 + 2.0 ** -11) * np.sign(W.ravel()[::7])   # ties: away from zero
        layers.append((W, None if i in no_bias else rng.normal(0, 1, c).astype(np.float32), True))
        c_in = c
    return layers


def on_gpu(layers):
    return [(torch.from_numpy(W).cuda(), None if b is None else torch.from_numpy(b).cuda(), r) for W, b, r in layers]


def check(packed, parts):
    want = np.concatenate(parts).view(np.uint32)
    got = packed.packed.cpu().numpy().view(np.uint32)
    assert got.shape == want.shape
    assert np.array_equal(got, want), np.flatnonzero(got != want)[:10]


def test_pointwise_mlp_segments_and_interpolated_source():
    rng = np.random.default_rng(1)
    spec = [(5, 0, 0), (12, 40, 3), (9, 0, 0), (20, 64, 8)]
    layers = random_layers(rng, 46, [20, 7, 33], no_bias=(1,))
    W1 = layers[0][0]
    Cpad0 = pad(20, 16)
    cols = np.cumsum([0] + [c for c, _, _ in spec])
    interp = [a_frag(W1[:, cols[s]:cols[s + 1]], pad(c, 8) // 8) for s, (c, M, _) in enumerate(spec) if M > 0]
    assert all(p.size == Cpad0 * pad(c, 8) for p, c in zip(interp, (12, 20)))
    dense = np.concatenate([W1[:, cols[s]:cols[s + 1]] for s, (_, M, _) in enumerate(spec) if M == 0], axis=1)
    parts = interp + [a_frag(dense, pad(14, 8) // 8), bias(layers[0][1], 20)] + chain(layers[1:], Cpad0)
    check(point_ops.pack_pointwise_mlp(spec, on_gpu(layers)), parts)


def test_knn_fusion_split_layer():
    rng = np.random.default_rng(2)
    C = 6
    before = random_layers(rng, 3 + C, [13, 10])
    after = random_layers(rng, 20, [17, 5], no_bias=(0,))
    W = after[0][0]                                          # [W_p | W_x]: the max half first
    parts = chain(before, pad(3 + C, 8))
    parts += [a_frag(W[:, 10:], pad(10, 16) // 8), bias(after[0][1], 17)] + chain(after[1:], pad(17, 16))
    parts.append(transposed(W[:, :10], pad(17, 16)))
    check(point_ops.pack_knn_fusion(C, on_gpu(before), on_gpu(after)), parts)


def test_pointwise_mlp_max_chain():
    rng = np.random.default_rng(3)
    layers = random_layers(rng, 11, [19, 6, 40], no_bias=(2,))
    check(point_ops.pack_pointwise_mlp_max(11, on_gpu(layers)), chain(layers, pad(11, 8)))


def test_node_mlp_per_sample_sources_between_dense_ones():
    rng = np.random.default_rng(4)
    spec = [(6, False), (5, True), (3, True), (7, False)]
    layers = random_layers(rng, 21, [21, 18])
    W1 = layers[0][0]
    Cpad0 = pad(21, 16)
    cols = np.cumsum([0] + [c for c, _ in spec])
    dense = np.concatenate((W1[:, 0:6], W1[:, 14:21]), axis=1)
    parts = [a_frag(dense, pad(13, 8) // 8), bias(layers[0][1], 21)] + chain(layers[1:], Cpad0)
    parts += [transposed(W1[:, cols[s]:cols[s + 1]], Cpad0) for s, (_, bc) in enumerate(spec) if bc]
    check(point_ops.pack_node_mlp(spec, on_gpu(layers)), parts)
