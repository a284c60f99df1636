"""point_ops.point_chain (DESIGN.md 4.34) on the device: the three per-point chains at the shipped widths against a
float64 torch restatement that uses the same dropout masks (outputs, running statistics, num_batches_tracked and
every gradient), bit-identical reruns, eval mode against the model's layers, the dropout stream, a captured fused
training step against the eager one, and peak memory of the KITTI head against the torch layers."""
import numpy as np
import pytest
import torch

from deepi2p_b200 import network, point_ops, synthetic, train

pytestmark = pytest.mark.gpu
TOL = 2.0 ** -10


def _pointnet(c_in, c_outs, last, dropouts=None, seed=0):
    torch.manual_seed(seed)
    pn = network._PointNet(c_in, c_outs, last, 0.1, dropouts).cuda()
    with torch.no_grad():                    # non-trivial BN parameters and running statistics
        for layer in pn.layers:
            if layer.norm is not None:
                C = layer.conv.out_channels
                layer.norm.weight.copy_(torch.rand(C) + 0.5)
                layer.norm.bias.copy_(torch.randn(C) * 0.1)
                layer.norm.running_mean.copy_(torch.randn(C) * 0.1)
                layer.norm.running_var.copy_(torch.rand(C) + 0.5)
            layer.conv.bias.copy_(torch.randn(layer.conv.out_channels) * 0.1)
    return pn


def _reference(sources, pn, state, add=None, in_col=0):
    """float64 train-mode chain with point_chain's masks; returns (out, {name: grad fn inputs}, running stats)."""
    x = torch.cat([s.double() for s in sources], dim=1)
    params, run, inter = [], [], []
    for l, layer in enumerate(pn.layers):
        W = layer.conv.weight.detach().double()[:, :, 0].clone().requires_grad_()
        b = layer.conv.bias.detach().double().clone().requires_grad_()
        Wu = W[:, in_col:in_col + x.shape[1]] if l == 0 else W
        y = torch.einsum("ck,bkn->bcn", Wu, x) + b[None, :, None]
        if l == 0 and add is not None:
            y = y + add
        y.retain_grad()
        inter.append({"x": x.detach(), "y": y, "W": Wu.detach()})
        p = [W, b]
        if layer.norm is not None:
            norm = layer.norm
            g = norm.weight.detach().double().clone().requires_grad_()
            be = norm.bias.detach().double().clone().requires_grad_()
            mean, var = y.mean(dim=(0, 2)), y.var(dim=(0, 2), unbiased=False)
            M = y.shape[0] * y.shape[2]
            run.append(((1 - norm.momentum) * norm.running_mean.double() + norm.momentum * mean.detach(),
                        (1 - norm.momentum) * norm.running_var.double() + norm.momentum * var.detach() * M / (M - 1)))
            invstd = 1 / torch.sqrt(var + norm.eps)
            xhat = (y - mean[None, :, None]) * invstd[None, :, None]
            z = xhat * g[None, :, None] + be[None, :, None]
            z.retain_grad()
            keep = (z > 0).double()
            y = torch.relu(z)
            if layer.dropout is not None:
                mask = point_ops.point_chain_dropout_mask(state, l, layer.dropout.p, *y.shape).double()
                y = y * mask / (1 - layer.dropout.p)
                keep = keep * mask / (1 - layer.dropout.p)
            inter[-1].update(z=z, xhat=xhat.detach(), keep=keep, k1=(g * invstd).detach())
            p += [g, be]
        else:
            run.append(None)
        params.append(p)
        x = y
    return x, params, run, inter


def _abs_backward(inter, gout):
    """The backward with every term replaced by its magnitude: per layer the scale of dY (`gy`) and of dZ (`gz`), and
    the scale of the sources' gradient.  A computed gradient's rounding error, the TF32 error of every layer above it
    included, is bounded by 2^-10 times a small multiple of these sums of |terms|."""
    a = gout.abs()
    for it in reversed(inter):
        if "keep" in it:
            gz = a * it["keep"]
            it["gz_abs"] = gz
            M = gz.shape[0] * gz.shape[2]
            xa = it["xhat"].abs()
            it["gy_abs"] = it["k1"].abs()[None, :, None] * (gz + gz.sum(dim=(0, 2), keepdim=True) / M
                                                          + xa * (gz * xa).sum(dim=(0, 2), keepdim=True) / M)
        else:
            it["gy_abs"] = a
        a = torch.einsum("ck,bcn->bkn", it["W"].abs(), it["gy_abs"])
    return a


def _check(got, want, scale, what, c=16):
    err = (got.double() - want).abs().max().item()
    bound = c * TOL * scale
    assert err <= bound, f"{what}: max error {err:.3e} > {bound:.3e}"


def _check_sum(got, want, scale, what, c=16, frac=0.0):
    """|got - want| <= c 2^-10 scale elementwise, with scale the sum of |terms| of each element (the form of
    test_pointwise_mlp_gpu.py's bound), for all but a share `frac` of the elements: a ReLU whose input is within TF32
    rounding of 0 can switch sides between the two computations and change single elements of a point-wise gradient
    completely."""
    bad = ((got.double() - want).abs() > c * TOL * scale).double().mean().item()
    assert bad <= frac, f"{what}: {bad:.2e} of the elements exceed c 2^-10 sum|terms|"


# (name, c_in, widths, norm_act_at_last, dropouts, sources' widths, in_col, add)
CHAINS = [("first", 7, [32, 32, 32], True, None, (3, 1, 3)),
          ("second", 64, [64, 64], True, None, (32, 32)),
          ("head_kitti", 736, [256, 256, 82], False, [0.5, 0.5, 0], (32, 64)),
          ("head_oxford", 736, [256, 256, 242], False, [0.5, 0.5, 0], (32, 64)),
          ("head_nuscenes", 736, [256, 256, 52], False, [0.5, 0.5, 0], (32, 64)),
          ("head_coarse", 736, [128, 128, 2], False, [0.5, 0.5, 0], (32, 64))]


def _case(spec, B=2, N=4096, seed=0):
    name, c_in, widths, last, drops, src_w = spec
    pn = _pointnet(c_in, widths, last, drops, seed)
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    sources = [torch.randn((B, c, N), device="cuda", generator=g).requires_grad_() for c in src_w]
    add, in_col = None, 0
    if sum(src_w) < c_in:
        in_col = c_in - sum(src_w)
        add = (torch.randn((B, widths[0], N), device="cuda", generator=g) * 2).requires_grad_()
    return pn, sources, add, in_col


@pytest.mark.parametrize("spec", CHAINS, ids=[c[0] for c in CHAINS])
def test_chain_matches_float64_reference(spec):
    _compare(spec, 2, 4096)


# point counts off the 64-point tile and the 32-point dW chunk, one sample, and 300 source rows (the input gradient
# then takes two blocks of output rows)
TAILS = [(CHAINS[2], 1, 1000), (CHAINS[1], 3, 4133), (CHAINS[0], 2, 77),
         (("wide", 300, [64, 16], False, None, (200, 100)), 2, 777)]


@pytest.mark.parametrize("spec, B, N", TAILS, ids=["head_B1_N1000", "second_N4133", "first_N77", "wide_sources"])
def test_chain_tails_single_sample_and_wide_sources(spec, B, N):
    _compare(spec, B, N)


def _compare(spec, B, N):
    pn, sources, add, in_col = _case(spec, B=B, N=N)
    state = point_ops.new_dropout_state(123, "cuda")
    used = state.clone()
    before = [(l.norm.running_mean.clone(), l.norm.running_var.clone(), l.norm.num_batches_tracked.clone())
              if l.norm is not None else None for l in pn.layers]
    out = point_ops.point_chain(sources, list(pn.layers), True, state, add=add, in_col=in_col)
    assert state[1].item() == used[1].item() + (1 if spec[4] else 0)
    g = torch.Generator(device="cuda").manual_seed(9)
    gout = torch.randn(out.shape, device="cuda", generator=g)
    out.backward(gout)

    for layer, bf in zip(pn.layers, before):
        if bf is not None:                      # the reference's update starts from the same buffers
            layer.norm.running_mean.data, bf_m = bf[0], layer.norm.running_mean.data
            layer.norm.running_var.data, bf_v = bf[1], layer.norm.running_var.data
            layer._got = (bf_m, bf_v, layer.norm.num_batches_tracked.clone())
            assert layer.norm.num_batches_tracked.item() == bf[2].item() + 1
    srcs = [s.detach().double().requires_grad_() for s in sources]
    add64 = add.detach().double().requires_grad_() if add is not None else None
    ref, params, run, inter = _reference(srcs, pn, used, add64, in_col)
    ref.backward(gout.double())
    src_abs = _abs_backward(inter, gout.double())

    scale = ref.abs().max().item()
    _check(out, ref, scale, "output")
    for l, (layer, p, r) in enumerate(zip(pn.layers, params, run)):
        W_g, b_g = layer.conv.weight.grad[:, :, 0], layer.conv.bias.grad
        it = inter[l]
        gy = it["gy_abs"]
        full = torch.einsum("bcn,bkn->ck", gy, it["x"].abs())
        Wsum = torch.zeros_like(p[0].grad)
        K = it["x"].shape[1]
        c0 = in_col if l == 0 else 0
        Wsum[:, c0:c0 + K] = full
        _check_sum(W_g, p[0].grad, Wsum, f"layer {l} dW", frac=1e-3)
        _check_sum(b_g, p[1].grad, gy.sum(dim=(0, 2)), f"layer {l} db")
        if r is not None:
            gz = it["gz_abs"]
            _check_sum(layer.norm.weight.grad, p[2].grad, (gz * it["xhat"].abs()).sum(dim=(0, 2)), f"layer {l} dgamma")
            _check_sum(layer.norm.bias.grad, p[3].grad, gz.sum(dim=(0, 2)), f"layer {l} dbeta")
            m, v, _ = layer._got
            _check(m, r[0], r[0].abs().max().item(), f"layer {l} running_mean")
            _check(v, r[1], r[1].abs().max().item(), f"layer {l} running_var")
    gy0, xs = inter[0]["gy_abs"], src_abs
    r = 0
    for s, s64 in zip(sources, srcs):
        # one flipped ReLU among a point's C_out channels changes every source row of that point
        _check_sum(s.grad, s64.grad, xs[:, r:r + s.shape[1]], "source grad", frac=1e-2)
        r += s.shape[1]
    if add is not None:
        # likewise one flipped ReLU of layer 2 at a point changes that point's whole dY column of layer 1
        _check_sum(add.grad, add64.grad, gy0, "add grad", frac=1e-2)


def _run_once(spec, seed=0):
    pn, sources, add, in_col = _case(spec, seed=seed)
    state = point_ops.new_dropout_state(5, "cuda")
    out = point_ops.point_chain(sources, list(pn.layers), True, state, add=add, in_col=in_col)
    out.backward(torch.ones_like(out))
    res = [out.detach()] + [s.grad for s in sources] + ([add.grad] if add is not None else [])
    for layer in pn.layers:
        res += [p.grad for p in layer.parameters()] + [b.clone() for b in layer.buffers()]
    return res


@pytest.mark.parametrize("spec", [CHAINS[1], CHAINS[2]], ids=["second", "head_kitti"])
def test_two_runs_are_bit_identical(spec):
    a, b = _run_once(spec), _run_once(spec)
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


def test_dropout_kept_fraction_and_new_masks_per_call():
    state = point_ops.new_dropout_state(77, "cuda")
    m0 = point_ops.point_chain_dropout_mask(state, 0, 0.5, 8, 256, 2048)
    n = m0.numel()
    kept = m0.double().mean().item()
    assert abs(kept - 0.5) <= 6 * (0.25 / n) ** 0.5
    state[1] += 1
    m1 = point_ops.point_chain_dropout_mask(state, 0, 0.5, 8, 256, 2048)
    assert abs(m1.double().mean().item() - 0.5) <= 6 * (0.25 / n) ** 0.5
    assert 0.4 < (m0 != m1).double().mean().item() < 0.6
    m2 = point_ops.point_chain_dropout_mask(state, 1, 0.5, 8, 256, 2048)
    assert 0.4 < (m1 != m2).double().mean().item() < 0.6


def test_captured_chain_draws_new_masks_on_every_replay():
    pn, sources, add, in_col = _case(CHAINS[2])
    state = point_ops.new_dropout_state(3, "cuda")
    src = [s.detach() for s in sources]
    a = add.detach()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        point_ops.point_chain(src, list(pn.layers), True, state, add=a, in_col=in_col)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = point_ops.point_chain(src, list(pn.layers), True, state, add=a, in_col=in_col)
    outs = []
    for _ in range(3):
        g.replay()
        outs.append(out.clone())
    torch.cuda.synchronize()
    assert not torch.equal(outs[0], outs[1]) and not torch.equal(outs[1], outs[2])
    assert state[1].item() == 4            # one eager call and three replays; capturing runs nothing


def _inputs(S, seed):
    rng = np.random.default_rng(seed)
    smps = [synthetic.make_sample(seed + s, 20480, "kitti") for s in range(S)]
    pc = torch.from_numpy(np.stack([s["points"] for s in smps])).cuda()
    idx = torch.from_numpy(np.stack([rng.permutation(20480)[:256] for _ in range(S)])).cuda()
    nodes = torch.gather(pc, 2, idx.unsqueeze(1).expand(S, 3, 256))
    return dict(pc=pc, intensity=torch.from_numpy(rng.random((S, 1, 20480), dtype=np.float32)).cuda(),
                sn=torch.from_numpy(rng.standard_normal((S, 3, 20480), dtype=np.float32)).cuda(),
                node_a=nodes[:, :, :128].contiguous(), node_b=nodes[:, :, 128:].contiguous(),
                img=torch.from_numpy(rng.random((S, 3, 160, 512), dtype=np.float32)).cuda(),
                K=torch.from_numpy(np.stack([s["K"] for s in smps])).float().cuda(),
                P=torch.from_numpy(np.stack([s["P_gt"][:3] for s in smps])).float().cuda())


def _model(point_layers, fine=True):
    m = network.KeypointDetector(**network.SHAPES["kitti"], fine=fine, point_layers=point_layers)
    m.load_state_dict(synthetic.seeded_state_dict(m, 1))
    return m.cuda()


@pytest.mark.parametrize("fine", [True, False])
def test_eval_mode_matches_the_torch_layers(fine):
    inp = _inputs(2, 40)
    args = [inp[k] for k in ("pc", "intensity", "sn", "node_a", "node_b", "img")]
    a, b = _model("torch", fine).eval(), _model("fused", fine).eval()
    with torch.no_grad():
        ra, rb = a(*args), b(*args)
    ra, rb = (ra, rb) if fine else ((ra,), (rb,))
    for x, y in zip(ra, rb):
        scale = x.abs().max().item()
        assert (x - y).abs().max().item() <= 64 * TOL * scale


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


@pytest.mark.parametrize("fine", [True, False])
def test_train_mode_model_matches_the_torch_layers_without_dropout(fine):
    """The whole fused model in train mode against the torch layers, with dropout off so both compute the same
    function.  The scores agree closely.  The gradients are compared loosely: the max-pools route a gradient to a
    different point where rounding reorders near-equal features, and that reaches every chain (a wiring error would be
    of order one; the head's wiring is tested tightly with shared inputs below)."""
    inp = _inputs(2, 60)
    args = [inp[k] for k in ("pc", "intensity", "sn", "node_a", "node_b", "img")]
    models, outs = {}, {}
    for mode in ("torch", "fused"):
        m = _model(mode, fine).train()
        for pn in (m.per_point_pn,):
            for layer in pn.layers:
                layer.dropout = None
        scores = m(*args)
        scores = torch.cat(scores, dim=1) if fine else scores
        g = torch.Generator(device="cuda").manual_seed(4)
        (scores * torch.randn(scores.shape, device="cuda", generator=g)).sum().backward()
        models[mode], outs[mode] = m, scores.detach()
    t, f = models["torch"], models["fused"]
    assert _rel(outs["fused"], outs["torch"]) < 2 ** -6
    chains = {"first": lambda m: m.pc_encoder.first_pointnet, "second": lambda m: m.pc_encoder.second_pointnet,
              "head": lambda m: m.per_point_pn}
    # first_pointnet and second_pointnet get much of their gradient through cluster_max_pool, whose arg-max moves to
    # another point where TF32 and cuDNN's rounding reorder near-equal features, so their gradients are compared
    # loosely (a wrong wiring would be of order one); the head's gradient does not pass through a max
    bound = {"first": 2 ** -1, "second": 2 ** -1, "head": 2 ** -1}
    for name, get in chains.items():
        for (k, pt), pf in zip(get(t).named_parameters(), get(f).parameters()):
            layer = get(t).layers[int(k.split(".")[1])]
            if k.endswith("conv.bias") and layer.norm is not None:
                continue                     # BatchNorm cancels the bias: its gradient is 0 plus rounding on both sides
            assert _rel(pf.grad, pt.grad) < bound[name], (name, k, _rel(pf.grad, pt.grad))
        for (k, bt), bf in zip(get(t).named_buffers(), get(f).buffers()):
            if bt.dtype == torch.int64:
                assert torch.equal(bt, bf), (name, k)
            else:
                assert _rel(bf, bt) < 2 ** -6, (name, k)
    wt, wf = t.per_point_pn.layers[0].conv.weight.grad[:, :, 0], f.per_point_pn.layers[0].conv.weight.grad[:, :, 0]
    for lo, hi in ((0, 128), (128, 640), (640, 736)):
        assert _rel(wf[:, lo:hi], wt[:, lo:hi]) < 2 ** -1, (lo, hi)


@pytest.mark.parametrize("fine", [True, False])
def test_fused_head_wiring_matches_the_torch_head(fine):
    """The head alone with identical inputs: KeypointDetector's fused head (pa / pb columns applied at the nodes, the
    dense sources from in_col) against per_point_pn over the 736-row cat, in train mode with dropout off.  With the
    inputs shared, only TF32 rounding separates them, so a shifted column split would show."""
    inp = _inputs(2, 70)
    pc, na, nb = inp["pc"], inp["node_a"], inp["node_b"]
    B, N = pc.shape[0], pc.shape[2]
    ia = point_ops.cluster_assign_forward(pc, na, k=3, want_centers=False)["min_k_idx"]
    ib = point_ops.cluster_assign_forward(pc, nb, k=3, want_centers=False)["min_k_idx"]
    g = torch.Generator(device="cuda").manual_seed(5)
    shared = [torch.randn(shape, device="cuda", generator=g)
              for shape in ((B, 128, 128), (B, 512, 128), (B, 32, N), (B, 64, N))]
    res = {}
    for mode in ("torch", "fused"):
        m = _model(mode, fine).train()
        for layer in m.per_point_pn.layers:
            layer.dropout = None
        upa, upb, f1, f2 = (t.clone().requires_grad_() for t in shared)
        if mode == "torch":
            pa = point_ops.upsample_by_interpolation(ia, pc, na, upa)
            pb = point_ops.upsample_by_interpolation(ib, pc, nb, upb)
            scores = m.per_point_pn(torch.cat((pa, pb, f1, f2), dim=1))
        else:
            scores = m._fused_head(pc, na, nb, ia, ib, upa, upb, f1, f2)
        gs = torch.Generator(device="cuda").manual_seed(6)
        (scores * torch.randn(scores.shape, device="cuda", generator=gs)).sum().backward()
        res[mode] = (scores.detach(), m, (upa.grad, upb.grad, f1.grad, f2.grad))
    (st, mt, it), (sf, mf, i_f) = res["torch"], res["fused"]
    assert _rel(sf, st) < 2 ** -6
    for name, a, b in zip(("up_node_a", "up_node_b", "first_pn_out", "second_pn_out"), i_f, it):
        assert _rel(a, b) < 2 ** -5, (name, _rel(a, b))
    for (k, pt), pf in zip(mt.per_point_pn.named_parameters(), mf.per_point_pn.parameters()):
        layer = mt.per_point_pn.layers[int(k.split(".")[1])]
        if k.endswith("conv.bias") and layer.norm is not None:
            continue
        assert _rel(pf.grad, pt.grad) < 2 ** -5, (k, _rel(pf.grad, pt.grad))
    wt = mt.per_point_pn.layers[0].conv.weight.grad[:, :, 0]
    wf = mf.per_point_pn.layers[0].conv.weight.grad[:, :, 0]
    for lo, hi in ((0, 128), (128, 640), (640, 736)):    # the pa, pb and dense column blocks separately
        assert _rel(wf[:, lo:hi], wt[:, lo:hi]) < 2 ** -5, (lo, hi)


def test_sources_changed_in_place_before_backward_raise():
    pn, sources, add, in_col = _case(CHAINS[1])
    x = sources[0] * 1.0
    out = point_ops.point_chain([x, sources[1]], list(pn.layers), True)
    with torch.no_grad():
        x.add_(1.0)
    with pytest.raises(RuntimeError, match="inplace"):
        out.sum().backward()


@pytest.mark.parametrize("C, K, M", [(256, 128, 128), (256, 512, 128), (300, 40, 77)])
def test_channel_product_matches_float64(C, K, M):
    g = torch.Generator(device="cuda").manual_seed(C + K)
    W = torch.randn((C, K), device="cuda", generator=g).requires_grad_()
    x = torch.randn((3, K, M), device="cuda", generator=g).requires_grad_()
    y = point_ops.channel_product(W, x)
    gy = torch.randn(y.shape, device="cuda", generator=g)
    y.backward(gy)
    W64, x64 = W.detach().double().requires_grad_(), x.detach().double().requires_grad_()
    ref = torch.einsum("ck,bkm->bcm", W64, x64)
    ref.backward(gy.double())
    _check_sum(y, ref, torch.einsum("ck,bkm->bcm", W64.detach().abs(), x64.detach().abs()), "out", c=4)
    _check_sum(W.grad, W64.grad, torch.einsum("bcm,bkm->ck", gy.double().abs(), x64.detach().abs()), "dW", c=4)
    _check_sum(x.grad, x64.grad, torch.einsum("ck,bcm->bkm", W64.detach().abs(), gy.double().abs()), "dx", c=4)
    first = (y.detach().clone(), W.grad.clone(), x.grad.clone())
    W.grad = x.grad = None
    y2 = point_ops.channel_product(W, x)
    y2.backward(gy)
    for u, v in zip(first, (y2.detach(), W.grad, x.grad)):
        assert torch.equal(u, v)


def _state(model, opt):
    out = {("model", k): v.clone() for k, v in model.state_dict().items()}
    for i, p in enumerate(model.parameters()):
        for k, v in opt.state[p].items():
            out[("adam", i, k)] = v.clone()
    return out


def test_captured_fused_step_is_the_eager_step_bit_for_bit():
    flags = torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark, \
        torch.are_deterministic_algorithms_enabled()
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    torch.use_deterministic_algorithms(True)
    try:
        batches = [_inputs(2, 100 + k) for k in range(6)]

        def run(capture):
            model = _model("fused")
            model.point_chain_state.copy_(point_ops.new_dropout_state(11, "cuda"))
            opt = train.make_optimizer(model)
            static = {k: torch.empty_like(v) for k, v in batches[0].items()}
            stats, losses = torch.zeros(5, device="cuda"), []
            torch.cuda.manual_seed(7)
            graph = None
            for k, b in enumerate(batches):
                for n, v in b.items():
                    static[n].copy_(v)
                if not capture or k < train.WARMUP_STEPS:
                    stats.copy_(train._stats(train.train_step(model, opt, static)))
                else:
                    if graph is None:
                        opt.zero_grad(set_to_none=True)
                        graph = torch.cuda.CUDAGraph()
                        with torch.cuda.graph(graph):
                            stats.copy_(train._stats(train.train_step(model, opt, static)))
                    graph.replay()
                losses.append(stats.clone())
            torch.cuda.synchronize()
            return _state(model, opt), torch.stack(losses), model.point_chain_state.clone()

        s_eager, l_eager, d_eager = run(False)
        s_graph, l_graph, d_graph = run(True)
        assert torch.equal(l_eager, l_graph)
        assert torch.equal(d_eager, d_graph)
        assert s_eager.keys() == s_graph.keys()
        bad = [k for k in s_eager if not torch.equal(s_eager[k], s_graph[k])]
        assert not bad, f"{len(bad)} tensors differ, first {bad[:3]}"
    finally:
        torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = flags[:2]
        torch.use_deterministic_algorithms(flags[2])


def _head_peak(mode, B=8, N=20480):
    torch.cuda.synchronize()
    pn = _pointnet(736, [256, 256, 82], False, [0.5, 0.5, 0])
    g = torch.Generator(device="cuda").manual_seed(3)
    f1 = torch.randn((B, 32, N), device="cuda", generator=g).requires_grad_()
    f2 = torch.randn((B, 64, N), device="cuda", generator=g).requires_grad_()
    upa = torch.randn((B, 128, 128), device="cuda", generator=g).requires_grad_()
    upb = torch.randn((B, 512, 128), device="cuda", generator=g).requires_grad_()
    pc = torch.randn((B, 3, N), device="cuda", generator=g)
    na, nb = pc[:, :, :128].contiguous(), pc[:, :, 128:256].contiguous()
    ia = point_ops.cluster_assign_forward(pc, na, k=3, want_centers=False)["min_k_idx"]
    ib = point_ops.cluster_assign_forward(pc, nb, k=3, want_centers=False)["min_k_idx"]
    state = point_ops.new_dropout_state(0, "cuda")
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    if mode == "torch":
        pa = point_ops.upsample_by_interpolation(ia, pc, na, upa)
        pb = point_ops.upsample_by_interpolation(ib, pc, nb, upb)
        out = pn(torch.cat((pa, pb, f1, f2), dim=1))
    else:
        W1 = pn.layers[0].conv.weight[:, :, 0]
        add = point_ops.upsample_by_interpolation(ia, pc, na, point_ops.channel_product(W1[:, :128], upa)) + \
            point_ops.upsample_by_interpolation(ib, pc, nb, point_ops.channel_product(W1[:, 128:640], upb))
        out = point_ops.point_chain([f1, f2], list(pn.layers), True, state, add=add, in_col=640)
    out.sum().backward()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def test_kitti_head_peak_memory_below_the_torch_layers():
    t, f = _head_peak("torch"), _head_peak("fused")
    assert f < 0.75 * t, (f, t)
