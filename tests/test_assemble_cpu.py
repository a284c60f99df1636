"""The batch-assembly oracle (oracle_assemble) against independent restatements, and host-side argument checks of
deepi2p_b200.assemble that run without a GPU."""
import ctypes
import math

import numpy as np
import pytest

import oracle_assemble as oa
from deepi2p_b200 import assemble, synthetic


def test_philox_known_answers():
    # Random123 kat_vectors, philox4x32 10 rounds
    cases = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
             ((0xffffffff,) * 4, (0xffffffff, 0xffffffff), (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
             ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
              (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]
    for ctr, key, want in cases:
        got = oa.philox4x32_10([np.array([c]) for c in ctr], key)[:, 0]
        assert tuple(int(v) for v in got) == want


class _RefFarthestSampler:
    """data/kitti_helper.py FarthestSampler, line by line (np.int -> np.int64)."""

    def __init__(self, dim=3):
        self.dim = dim

    def calc_distances(self, p0, points):
        return ((p0 - points) ** 2).sum(axis=0)

    def sample(self, pts, k):
        farthest_pts = np.zeros((self.dim, k))
        farthest_pts_idx = np.zeros(k, dtype=np.int64)
        init_idx = np.random.randint(len(pts))
        farthest_pts[:, 0] = pts[:, init_idx]
        farthest_pts_idx[0] = init_idx
        distances = self.calc_distances(farthest_pts[:, 0:1], pts)
        for i in range(1, k):
            idx = np.argmax(distances)
            farthest_pts[:, i] = pts[:, idx]
            farthest_pts_idx[i] = idx
            distances = np.minimum(distances, self.calc_distances(farthest_pts[:, i:i + 1], pts))
        return farthest_pts, farthest_pts_idx


def _fps_inputs(dim):
    rng = np.random.default_rng(dim)
    rand = rng.normal(0, 10, (dim, 700)).astype(np.float32)
    dup = np.repeat(rng.normal(0, 1, (dim, 40)).astype(np.float32), 5, axis=1)
    g = np.arange(8, dtype=np.float32)
    lat = np.stack(np.meshgrid(*([g] * dim), indexing="ij")).reshape(dim, -1)
    return [rand, dup, lat, rand.astype(np.float64)]


@pytest.mark.parametrize("dim", [2, 3])
def test_fps_oracle_matches_reference_sampler(dim):
    for pts in _fps_inputs(dim):
        for seed in range(3):
            np.random.seed(seed)
            ref_pts, ref_idx = _RefFarthestSampler(dim).sample(pts, 64)
            np.random.seed(seed)
            start = np.random.randint(len(pts))
            idx, nodes = oa.fps(pts, 64, start)
            assert np.array_equal(idx, ref_idx)
            assert np.array_equal(nodes.astype(np.float64), ref_pts)


@pytest.mark.parametrize("n", [1, 2, 20480 // 3, 20479, 20480, 20481, 40960])
def test_repeat_rule(n):
    N = 20480
    idx = oa.resample_index(n, N, 3, 11)
    assert idx.shape == (N,) and idx.min() >= 0 and idx.max() < n
    counts = np.bincount(idx, minlength=n)
    if n >= N:
        assert counts.max() == 1
    else:
        r = 1
        while (r + 1) * n < N:
            r += 1
        assert set(np.unique(counts)) <= {r, r + 1}
        tail = idx[r * n:]
        assert len(np.unique(tail)) == len(tail) == N - r * n
        assert np.array_equal(idx[:r * n], np.tile(np.arange(n), r))


def test_key_order_is_a_uniform_choice():
    # each position is equally likely to be drawn first (loose chi-square over 200 samples of 10 points)
    firsts = np.array([oa.key_order(10, s, oa.STREAM_RESAMPLE, 5)[0] for s in range(2000)])
    c = np.bincount(firsts, minlength=10)
    assert ((c - 200.0) ** 2 / 200.0).sum() < 40.0


def test_angles2rotation_matrix():
    rng = np.random.default_rng(0)
    ang = rng.uniform(-math.pi, math.pi, (5, 3))
    got = assemble.angles2rotation_matrix(ang)
    for a, R in zip(ang, got):
        Rx = np.array([[1, 0, 0], [0, np.cos(a[0]), -np.sin(a[0])], [0, np.sin(a[0]), np.cos(a[0])]])
        Ry = np.array([[np.cos(a[1]), 0, np.sin(a[1])], [0, 1, 0], [-np.sin(a[1]), 0, np.cos(a[1])]])
        Rz = np.array([[np.cos(a[2]), -np.sin(a[2]), 0], [np.sin(a[2]), np.cos(a[2]), 0], [0, 0, 1]])
        assert np.allclose(R, np.dot(Rz, np.dot(Ry, Rx)), atol=1e-15)


def test_compose_matches_the_oracle_and_matmul():
    rng = np.random.default_rng(1)
    A, B = rng.normal(size=(3, 4, 4)), rng.normal(size=(3, 4, 4))
    got = assemble.compose(A, B)
    for s in range(3):
        assert np.array_equal(got[s], oa.compose(A[s], B[s]))
        assert np.allclose(got[s], A[s] @ B[s], rtol=1e-14, atol=1e-14)


@pytest.mark.parametrize("shape", ["kitti", "oxford"])
def test_pose_composition_reprojects(shape):
    """P (assembled) applied to the assembled points projects to the pixels P_base pre gives the source points."""
    smp = synthetic.make_loader_sample(3, shape, n_rings=8, n_azimuth=64)
    args = assemble.kitti_args(smp["Pc"], smp["Pji"]) if shape == "kitti" else assemble.oxford_args(smp["P_cam_pc"])
    Pr, _ = assemble.random_transforms(4, "train", args["amplitudes"], rng=7, flip=args["flip"])
    x, _, _ = oa.accumulate(smp["frames"], smp["frame_T"])
    pre = np.asarray(args["pre"])
    for s in range(4):
        M = assemble.compose(Pr[s], pre)
        pc = oa.affine(M, x)
        P = assemble.compose(args["P_base"], assemble.rigid_inverse(Pr[s]))
        a = smp["K"] @ (P[:3, :3] @ pc.astype(np.float64) + P[:3, 3:])
        Pb = assemble.compose(args["P_base"], pre)
        b = smp["K"] @ (Pb[:3, :3] @ x.astype(np.float64) + Pb[:3, 3:])
        front = b[2] > 1.0
        ua, ub = a[:2, front] / a[2, front], b[:2, front] / b[2, front]
        scale = np.abs(x).max()
        assert np.abs(ua - ub).max() < 1e-4 * scale


def test_random_transforms_modes():
    Pr, flip = assemble.random_transforms(64, "train", (1.0, 0.5, 1.0, 0.0, 2 * math.pi, 0.0), rng=0)
    R = Pr[:, :3, :3]
    assert np.allclose(np.einsum("sji,sjk->sik", R, R), np.eye(3)[None], atol=1e-12)
    assert np.allclose(np.linalg.det(R), np.where(flip, -1.0, 1.0))
    assert 0 < flip.sum() < 64 and np.abs(Pr[:, 1, 3]).max() <= 0.5
    Pr, flip = assemble.random_transforms(8, "val_random_Ry", rng=0)
    assert not flip.any() and np.allclose(Pr[:, 1], [0, 1, 0, 0]) and np.allclose(Pr[:, :3, 3], 0)
    Pr, _ = assemble.random_transforms(3, "test")
    assert np.array_equal(Pr, np.tile(np.eye(4), (3, 1, 1)))
    with pytest.raises(ValueError):
        assemble.random_transforms(3, "bogus")


def test_host_rejection_without_gpu():
    from deepi2p_b200 import _native
    lib = _native.load()
    buf = ctypes.create_string_buffer(1024)
    a = ctypes.addressof(buf)
    # k > n_stride, k < 1, more than 65536 candidates
    assert lib.fps_batch_f32(a, None, 16, 1, 17, None, a, a, None) == -22
    assert lib.fps_batch_f64(a, None, 16, 1, 0, None, a, a, None) == -22
    assert lib.fps_batch_f32(a, None, 65537, 1, 4, None, a, a, None) == -22
    assert b"65536" in lib.dib_last_error()
    # 8 M > N
    assert lib.assemble_candidates_f32(a, 1024, 1, 0, 0, 1032, a, a, a, 1024, None) == -22
    # input_pt_num < 1
    assert lib.assemble_resample_f32(a, a, None, None, 16, 1, 0, 0, a, 0.01, 0.05, 0, a, a, None, a, a, 1024,
                                     None) == -22
    assert b"input_pt_num" in lib.dib_last_error()
    # workspace too small
    assert lib.assemble_accumulate_f32(a, a, None, None, 16, 1, a, a, 1, 0.0, a, a, None, 16, a, a, 16, None) == -22
    assert lib.assemble_accumulate_workspace_bytes(1, 16, 1) > 0
    with pytest.raises(ValueError):
        assemble.assemble_batch({}, "train", 0, input_pt_num=1000, node_a_num=128)
    with pytest.raises(ValueError):
        assemble.assemble_batch({}, "train", 0, input_pt_num=0)
