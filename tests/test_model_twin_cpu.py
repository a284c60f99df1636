"""A float64 twin of the reference classifier network (models/networks_united.py, networks_pc.py, layers_pc.py), written
out in plain torch from the reference's composition and independent of KeypointDetector.forward and point_ops, and
its check against the reference's own float64 run (tests/golden/network_small.npz) in train and eval mode.

The twin is a function of (parameters and buffers, inputs, image maps, decisions).  A decision is an integer choice the
network makes: the clustering and kNN searches and the arg-max of every max site.  Given decisions, every gather uses
them; without, the twin decides as the reference does (`DECISIONS`).  tests/test_model_twin_gpu.py runs the twin along
the decisions a fused training run recorded, so that what remains between the two is rounding; its magnitude run (the
same composition over |parameters| and |inputs|, BatchNorm + ReLU by their sum-of-|terms| backward) gives the per-element
gradient bounds there."""
import os

import numpy as np
import pytest
import torch

from deepi2p_b200 import network, synthetic

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "network_small.npz")
BN_EPS = 1e-5
# The reference's PointNets and whether their last layer has BatchNorm + ReLU (norm_act_at_last); every other layer has.
POINTNETS = {"pc_encoder.first_pointnet": True, "pc_encoder.second_pointnet": True,
             "pc_encoder.final_pointnet": True, "node_b_attention_pn": False, "node_b_pn": False,
             "node_a_attention_pn": False, "node_a_pn": False, "per_point_pn": False}
HEAD_DROPOUT = (0.5, 0.5, 0.0)              # per_point_pn's dropout_list
# Decision sites, and the rule by which the twin decides each when none is given:
#   pa, pb, ab                nearest nodes (pc -> node_a, pc -> node_b, node_a -> node_b), the top-k on (d^2, index);
#                             pa[..., 0] is the cluster assignment
#   knn                       the kNN module's K nearest cluster means of each node_b, the top-K on (d^2, index)
#   cluster_first, _second    the cluster max-pools: index_max's rule (the arg-max on the features cast to float32,
#                             lowest index on ties, index 0 when the segment's maximum is not above -1000)
#   knn_before, knn_after     the kNN module's maxes over K, and
#   global                    the max over the nodes: the float64 arg-max, lowest index on ties
DECISIONS = ("pa", "pb", "ab", "knn", "cluster_first", "cluster_second", "knn_before", "knn_after", "global")


class BnReluAbs(torch.autograd.Function):
    """The magnitude graph of train-mode BatchNorm + ReLU over [B, C, cols]: forward gives |a| of the value run,
    backward the sum of |terms| of the BatchNorm backward (dY = k1 (dZ - mean dZ - x^ mean(dZ x^))) and of dgamma,
    dbeta."""

    @staticmethod
    def forward(ctx, ya, ga, bea, a_abs, keep, xhat_abs, k1_abs):
        ctx.save_for_backward(keep, xhat_abs, k1_abs)
        return a_abs.clone()

    @staticmethod
    def backward(ctx, g):
        keep, xa, k1 = ctx.saved_tensors
        gz = g * keep
        M = gz.shape[0] * gz.shape[2]
        gy = k1[None, :, None] * (gz + gz.sum(dim=(0, 2), keepdim=True) / M
                                  + xa * (gz * xa).sum(dim=(0, 2), keepdim=True) / M)
        return gy, (gz * xa).sum(dim=(0, 2)), gz.sum(dim=(0, 2)), None, None, None, None


def first_argmax(x, dim):
    """The arg-max along dim, lowest index on ties (keepdim)."""
    n = torch.arange(x.shape[dim], device=x.device).reshape([-1 if d == dim % x.dim() else 1 for d in range(x.dim())])
    hit = x == x.amax(dim=dim, keepdim=True)
    return torch.where(hit, n, x.shape[dim]).amin(dim=dim, keepdim=True)


def top2_gap(x, dim):
    """Smallest relative gap between the largest and second-largest value along dim over the groups whose maximum is
    above 0 (a group whose maximum is a ReLU zero passes no gradient, whichever index it picks); inf without such."""
    if x.shape[dim] < 2:
        return float("inf")
    v = x.topk(2, dim=dim).values
    v0, v1 = v.select(dim, 0), v.select(dim, 1)
    live = v0 > 0
    return float(((v0 - v1) / v0)[live].min()) if live.any() else float("inf")


def index_max_rule(f32, min_idx, M):
    """index_max's arg-max: for each (b, c, m), the lowest n with min_idx[b, n] == m attaining the segment's maximum of
    f32[b, c, :], if that maximum is above -1000, else 0.  Returns (sel [B,C,M] int64, relative top-2 gap of the
    segments whose maximum is above 0)."""
    B, C, N = f32.shape
    seg = min_idx[:, None, :].expand(B, C, N)
    mx = torch.full((B, C, M), -float("inf"), dtype=f32.dtype, device=f32.device)
    mx = mx.scatter_reduce(2, seg, f32, "amax")
    hit = f32 == mx.gather(2, seg)
    n = torch.arange(N, device=f32.device).expand(B, C, N)
    first = torch.full((B, C, M), N, dtype=torch.int64, device=f32.device)
    first = first.scatter_reduce(2, seg, torch.where(hit, n, N), "amin")
    sel = torch.where(mx > -1000, first, 0)
    rest = f32.clone()
    rest.scatter_(2, sel, -float("inf"))                  # the chosen point out, its segment's runner-up remains
    second = torch.full_like(mx, -float("inf")).scatter_reduce(2, seg, rest, "amax")
    live = (mx > 0) & (second > -float("inf"))
    gap = float(((mx - second) / mx)[live].min()) if live.any() else float("inf")
    return sel, gap


def nearest(q, d, k):
    """The k nearest of d [B,3,M] to each of q [B,3,Nq], nearest first, on (d^2, index): [B,Nq,k] int64, and the
    smallest relative gap between consecutive squared distances up to the (k+1)-th."""
    d2 = ((q[:, :, :, None] - d[:, :, None, :]) ** 2).sum(1)
    s, i = torch.sort(d2, dim=2, stable=True)
    kk = min(k + 1, d2.shape[2])
    gap = float(((s[..., 1:kk] - s[..., :kk - 1]) / s[..., 1:kk]).min()) if kk > 1 else float("inf")
    return i[..., :k].contiguous(), gap


def _gather_cols(f, idx):
    """f [B,C,M] at idx [B,Nq,k] -> [B,C,Nq,k]."""
    B, C = f.shape[:2]
    return f.gather(2, idx.reshape(B, 1, -1).expand(B, C, -1)).reshape(B, C, *idx.shape[1:])


class Twin:
    """One run of the twin.  P: parameter and buffer name -> float64 tensor (the state_dict's names; parameters may be
    leaves that require grad).  dec: decisions by DECISIONS name (missing ones are decided here and added).  keep:
    per_point_pn layer name -> dropout keep mask [B,C,N] (1 = kept) or None (dropout off).  mag: None for a value run,
    or the value run (a Twin) whose decisions, dropout masks and BatchNorm state a magnitude run follows; P then holds
    |parameters| and the inputs their magnitudes.  After `scores`, `running` holds the running statistics the
    train-mode BatchNorm layers write (name -> tensor), `margins` the top-2 gaps of the sites decided here and `maxima`
    the values the group maxes took."""

    def __init__(self, P, train=True, dec=None, keep=None, mag=None, momentum=0.1, k_ab=16, k_interp=3):
        self.P, self.train, self.keep, self.mag = P, train, keep, mag
        self.dec = dict(mag.dec if mag is not None else (dec or {}))
        self.momentum, self.k_ab, self.k_interp = momentum, k_ab, k_interp
        self.bn, self.running, self.margins, self.maxima = {}, {}, {}, {}
        assert mag is None or train, "the magnitude graph is that of train-mode BatchNorm"

    def const(self, t):
        """A tensor that enters the graph as data (coordinates, masks, weights): its magnitude in a magnitude run."""
        return t.abs() if self.mag is not None else t

    def layer(self, name, x, norm, p):
        P = self.P
        W = P[name + ".conv.weight"]
        W = W.reshape(W.shape[0], -1)
        B, C = x.shape[:2]
        y = torch.einsum("ck,bkn->bcn", W, x.reshape(B, C, -1)) + P[name + ".conv.bias"][None, :, None]
        if norm:
            g, be = P[name + ".norm.weight"], P[name + ".norm.bias"]
            rm, rv = P[name + ".norm.running_mean"], P[name + ".norm.running_var"]
            if self.mag is not None:
                y = BnReluAbs.apply(y, g, be, *self.mag.bn[name])
            else:
                if self.train:
                    mean, var = y.mean(dim=(0, 2)), y.var(dim=(0, 2), unbiased=False)
                    n, m = y.shape[0] * y.shape[2], self.momentum
                    self.running[name + ".norm.running_mean"] = (1 - m) * rm + m * mean.detach()
                    self.running[name + ".norm.running_var"] = (1 - m) * rv + m * var.detach() * n / (n - 1)
                else:
                    mean, var = rm, rv
                invstd = 1 / torch.sqrt(var + BN_EPS)
                xhat = (y - mean[None, :, None]) * invstd[None, :, None]
                z = xhat * g[None, :, None] + be[None, :, None]
                y = torch.relu(z)
                self.bn[name] = (y.detach().abs(), (z > 0).to(z.dtype).detach(), xhat.detach().abs(),
                                 (g * invstd).detach().abs())
            if p > 0 and self.train and self.keep is not None:
                y = y * self.const(self.keep[name].to(y.dtype) / (1 - p))
        return y.reshape(B, -1, *x.shape[2:])

    def pointnet(self, prefix, x):
        n = sum(1 for k in self.P if k.startswith(prefix + ".layers.") and k.endswith(".conv.weight"))
        for i in range(n):
            p = HEAD_DROPOUT[i] if prefix == "per_point_pn" else 0.0
            x = self.layer(f"{prefix}.layers.{i}", x, POINTNETS[prefix] or i < n - 1, p)
        return x

    def search(self, site, q, d, k):
        if site not in self.dec:
            self.dec[site], self.margins[site] = nearest(q, d, k)
        return self.dec[site]

    def group_max(self, site, x, dim):
        if site not in self.dec:
            self.dec[site], self.margins[site] = first_argmax(x.detach(), dim), top2_gap(x.detach(), dim)
        out = x.gather(dim, self.dec[site])
        self.maxima[site] = out.detach()
        return out

    def cluster_max(self, site, f, min_idx, M, mask):
        if site not in self.dec:
            self.dec[site], self.margins[site] = index_max_rule(f.detach().float(), min_idx, M)
        return f.gather(2, self.dec[site]) * self.const(mask)[:, None, :]

    def interpolate(self, site, q, nodes, f):
        """Inverse-distance interpolation of node features f [B,C,M] onto q [B,3,Nq] over the site's k nearest nodes:
        w_j = 1 - d_j / sum_j d_j, out = sum_j w_j f[idx_j]."""
        idx = self.search(site, q, nodes, self.k_interp)
        d = (q[:, :, :, None] - _gather_cols(nodes, idx)).norm(dim=1)
        w = self.const(1 - d / d.sum(dim=2, keepdim=True))
        return (w[:, None] * _gather_cols(f, idx)).sum(dim=3)

    @staticmethod
    def attend(fmap, att):
        """torch.mean(F.unsqueeze(3) * att.unsqueeze(1), dim=2) with F the map viewed [B,C,P]."""
        F = fmap.reshape(fmap.shape[0], fmap.shape[1], -1)
        return torch.einsum("bcp,bpm->bcm", F, att) / F.shape[2]

    def scores(self, pc, intensity, sn, node_a, node_b, s16, s32, img_global=None):
        """Inputs float64 [B,3,N], [B,1,N], [B,3,N], [B,3,Ma], [B,3,Mb]; the image maps s16 [B,256,h,w], s32
        [B,512,h',w'] and optionally img_global [B,512] (else the mean of s32 over its pixels).  In a magnitude run
        all of them are magnitudes except the coordinates, which stay the values.  Returns [B, 2 (+ L), N]."""
        B, N, Ma, Mb = pc.shape[0], pc.shape[2], node_a.shape[2], node_b.shape[2]
        # PCEncoder: clusters of the nearest node_a, decentred points, two PointNets with a cluster max-pool each
        pa = self.search("pa", pc, node_a, self.k_interp)
        min_idx = pa[:, :, 0]
        onehot = torch.zeros((B, N, Ma), dtype=pc.dtype, device=pc.device).scatter_(2, min_idx[:, :, None], 1.0)
        count = onehot.sum(dim=1)                                               # [B,Ma]
        mask = (count > 0).to(pc.dtype)
        # the reference's point counts are float32 (networks_pc.py:71-76), so count + 1e-5 is rounded to float32
        denom = (count.float() + 1e-5).to(pc.dtype)
        cluster_mean = torch.einsum("bcn,bnm->bcm", pc, onehot) / denom[:, None, :]
        pc_dec = pc - cluster_mean.gather(2, min_idx[:, None, :].expand(B, 3, N))
        first = self.pointnet("pc_encoder.first_pointnet", torch.cat((self.const(pc_dec), intensity, sn), dim=1))
        first_max = self.cluster_max("cluster_first", first, min_idx, Ma, mask)
        scattered = first_max.gather(2, min_idx[:, None, :].expand(B, first.shape[1], N))
        second = self.pointnet("pc_encoder.second_pointnet", torch.cat((first, scattered), dim=1))
        node_a_features = self.cluster_max("cluster_second", second, min_idx, Ma, mask)
        # GeneralKNNFusionModule: query node_b, database the cluster means and node_a_features
        knn = self.search("knn", node_b, cluster_mean, self.k_ab)               # [B,Mb,K]
        coords = _gather_cols(cluster_mean, knn) - node_b[:, :, :, None]
        x = torch.cat((self.const(coords), _gather_cols(node_a_features, knn)), dim=1)
        for i in range(2):
            x = self.layer(f"pc_encoder.knnlayer.layers_before.{i}", x, True, 0.0)
        pooled = self.group_max("knn_before", x, 3)
        y = torch.cat((pooled.expand_as(x), x), dim=1)
        for i in range(2):
            y = self.layer(f"pc_encoder.knnlayer.layers_after.{i}", y, True, 0.0)
        node_b_features = self.group_max("knn_after", y, 3).squeeze(3)        # [B,Cb,Mb]
        final = self.pointnet("pc_encoder.final_pointnet", torch.cat((self.const(node_b), node_b_features), dim=1))
        global_feature = self.group_max("global", final, 2)                    # [B,Cg,1]
        # image: the stride-16 and stride-32 maps and the global feature, expanded over the nodes
        if img_global is None:
            img_global = s32.mean(dim=(2, 3))
        ig_b, ig_a = img_global[:, :, None].expand(-1, -1, Mb), img_global[:, :, None].expand(-1, -1, Ma)
        att_b = self.pointnet("node_b_attention_pn", torch.cat((node_b_features, ig_b), dim=1))
        up_node_b = self.pointnet("node_b_pn", torch.cat((node_b_features, global_feature.expand(-1, -1, Mb),
                                                          self.attend(s32, att_b), ig_b), dim=1))
        interp_pb = self.interpolate("pb", pc, node_b, up_node_b)
        att_a = self.pointnet("node_a_attention_pn", torch.cat((node_a_features, ig_a), dim=1))
        interp_ab = self.interpolate("ab", node_a, node_b, up_node_b)
        up_node_a = self.pointnet("node_a_pn", torch.cat((node_a_features, interp_ab, self.attend(s16, att_a)), dim=1))
        interp_pa = self.interpolate("pa", pc, node_a, up_node_a)
        return self.pointnet("per_point_pn", torch.cat((interp_pa, interp_pb, first, second), dim=1))


def state64(model, requires_grad=True):
    """The model's point-side parameters and buffers as float64 copies (parameters as leaves that require grad); the
    image encoder's are left out, since it runs as a module (or is replaced by its maps)."""
    params = {k for k, _ in model.named_parameters()}
    return {k: v.detach().double().clone().requires_grad_(requires_grad and k in params)
            for k, v in model.state_dict().items() if not k.startswith("img_encoder.")
            and not k.endswith("num_batches_tracked")}


# ------------------------------------------------------------------------------------------------------------------
# against the reference's own float64 network

# The golden's scores and kept gradient entries against the twin's: max |twin - golden| / max |golden|.  Both are
# float64 runs of the same composition with different summation orders (einsum against conv1d, the twin's ResNet copy
# against the reference's), so they agree to far below this.
REL = 1e-9


@pytest.fixture(scope="module")
def golden():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


@pytest.fixture
def no_project_forward(monkeypatch):
    """The twin runs without KeypointDetector.forward and without any point_ops function."""
    from deepi2p_b200 import point_ops

    def refuse(*args, **kwargs):
        raise AssertionError("the twin reached KeypointDetector.forward or a point_ops function")
    monkeypatch.setattr(network.KeypointDetector, "forward", refuse)
    for name in dir(point_ops):
        if callable(getattr(point_ops, name)) and not name.startswith("__"):
            monkeypatch.setattr(point_ops, name, refuse)


def _small_run(golden, train):
    """The golden's model and inputs through the twin on the CPU, with its own decisions, dropout off.  Returns (twin,
    coarse, fine, {golden grad key: float64 gradient})."""
    g = golden
    B, N, Ma, Mb, H, W = 2, 2048, 128, 128, 64, 128
    model = network.KeypointDetector(img_H=H, img_W=W, node_a_num=Ma, node_b_num=Mb)
    model.load_state_dict(synthetic.seeded_state_dict(model, int(g["weight_seed"])), strict=True)
    inp = synthetic.make_network_inputs(int(g["input_seed"]), B, N, Ma, Mb, H, W, 8)
    sums = np.array([inp[k].astype(np.float64).sum() for k in g["input_names"]])
    assert np.array_equal(sums, g["input_sums"]), "synthetic.make_network_inputs no longer gives the golden's inputs"
    x = {k: torch.from_numpy(v).double() for k, v in inp.items()}
    P = state64(model)
    backbone = model.img_encoder.backbone.double().train(train)
    s16, s32 = backbone(x["img"])
    t = Twin(P, train=train)
    scores = t.scores(x["pc"], x["intensity"], x["sn"], x["node_a"], x["node_b"], s16, s32)
    grads = {}
    if train:
        ((scores[:, :2] * x["lw_coarse"]).sum() + (scores[:, 2:] * x["lw_fine"]).sum()).backward()
        named = dict(model.named_parameters())
        for i, k in enumerate(g["grad_keys"]):
            grad = named[k].grad if k.startswith("img_encoder.") else P[k].grad
            grads[i] = grad.reshape(-1)[::int(g["grad_stride"][i])].numpy()
    return t, scores[:, :2].detach().numpy(), scores[:, 2:].detach().numpy(), grads


def _close(got, want, what):
    err = np.abs(got - want).max() / np.abs(want).max()
    print(f"{what}: max |twin - reference| {err:.2e} of max|reference|")
    assert err < REL, f"{what}: {err:.2e} of max|reference|"


def test_twin_matches_the_reference_network_in_train_mode(golden, no_project_forward):
    t, coarse, fine, grads = _small_run(golden, True)
    stride = int(golden["point_stride"])
    _close(coarse[..., ::stride], golden["train_coarse"], "train coarse")
    _close(fine[..., ::stride], golden["train_fine"], "train fine")
    for i, grad in grads.items():
        _close(grad, golden[f"grad_{i}"], f"grad {golden['grad_keys'][i]}")
    # every site was decided here, each with a margin far above float64 rounding: the golden's run and the twin's
    # cannot have decided one differently
    assert set(t.margins) == set(DECISIONS)
    print("decision margins (relative top-2 gap):", {k: f"{v:.2e}" for k, v in t.margins.items()})
    assert min(t.margins.values()) > 1e-9


def test_twin_matches_the_reference_network_in_eval_mode(golden, no_project_forward):
    t, coarse, fine, _ = _small_run(golden, False)
    stride = int(golden["point_stride"])
    _close(coarse[..., ::stride], golden["eval_coarse"], "eval coarse")
    _close(fine[..., ::stride], golden["eval_fine"], "eval fine")
    print("decision margins (relative top-2 gap):", {k: f"{v:.2e}" for k, v in t.margins.items()})
    assert min(t.margins.values()) > 1e-9


def test_index_max_rule_on_ties_empty_segments_and_the_floor():
    f = torch.tensor([[[1.0, 3.0, 3.0, 2.0, -2000.0, 5.0]]])
    min_idx = torch.tensor([[0, 0, 0, 1, 2, 1]])
    sel, _ = index_max_rule(f, min_idx, 4)
    # segment 0: tie at 3 -> the lower index 1; segment 1: 5 at index 5; segment 2: -2000 is not above -1000 -> 0;
    # segment 3 is empty -> 0
    assert sel.tolist() == [[[1, 5, 0, 0]]]


def test_given_decisions_are_followed():
    """A twin run given another run's decisions reproduces it exactly, and one given a different arg-max moves the
    scores: the gathers read the decisions, not a fresh arg-max."""
    torch.manual_seed(0)
    model = network.KeypointDetector(img_H=64, img_W=128, node_a_num=32, node_b_num=32, k_ab=4)
    inp = synthetic.make_network_inputs(3, 2, 256, 32, 32, 64, 128, 8)
    x = {k: torch.from_numpy(v).double() for k, v in inp.items()}
    s16, s32 = torch.rand(2, 256, 4, 8, dtype=torch.float64), torch.rand(2, 512, 2, 4, dtype=torch.float64)
    run = lambda dec: Twin(state64(model, False), dec=dec, k_ab=4).scores(
        x["pc"], x["intensity"], x["sn"], x["node_a"], x["node_b"], s16, s32)
    a = Twin(state64(model, False), k_ab=4)
    want = a.scores(x["pc"], x["intensity"], x["sn"], x["node_a"], x["node_b"], s16, s32)
    assert torch.equal(run(a.dec), want)
    moved = dict(a.dec, knn_after=(a.dec["knn_after"] + 1) % 4)
    assert not torch.allclose(run(moved), want)
