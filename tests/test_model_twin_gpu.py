"""KeypointDetector's training forward and backward in every point-layer mode against the float64 twin of the
reference network (tests/test_model_twin_cpu.py), run along the integer decisions the model's own run made.

Each case runs the model once in train mode, with every point_ops op that forward() calls wrapped to record its
arguments and results, and calls backward with a seeded random cotangent on the scores.  From the recording:
  - the clustering, the kNN grouping and the three interpolation searches: the recorded integer indices;
  - the cluster max-pools: index_max_forward on the recorded features (the rule cluster_max_pool follows);
  - point_branch's group maxes ("fused_all": the kNN module's two maxes over K and the global max over the nodes): the
    recorded call rerun with output="both" on a copy of its layers as they were before the call, then the first
    maximal index of each group; where those maxes are torch.max calls over a module's output ("fused"), a forward
    hook on that module gives the same;
  - the head's dropout masks: point_chain_dropout_mask on the dropout state recorded before the call.
The image branch stays with torch and cuDNN: its stride-16 and stride-32 maps enter both runs as the same leaves, and
the gradients reaching them and the global image feature are compared instead of cuDNN's weight gradients.

What remains between the two runs is rounding (TF32 products in the fused layers) and the occasional ReLU input within
rounding of zero, so the bounds are rounding bounds: the scores and running statistics within C_OUT u max|ref|, and
every point-layer parameter gradient and the three image-side gradients within C_GRAD u sum|terms| per element, sum|terms|
being the twin's magnitude run (the same composition over |parameters| and |inputs|), for all but a share FRAC of the
elements (a ReLU input that flips moves its element's whole gradient).  Every per-parameter relative 2-norm is also
bounded (BOUNDS says how tightly, and why the fused modes cannot be held far below the 2^-1 of the existing whole-model
tests).  The measured worst ratios are printed (pytest -s) and recorded beside the bounds."""
import copy
import inspect

import pytest
import torch

from deepi2p_b200 import network, point_ops, synthetic
from test_model_twin_cpu import DECISIONS, Twin, first_argmax, state64

pytestmark = pytest.mark.gpu

# (unit u, C_OUT, C_GRAD, FRAC, REL_GRAD) per mode.  The "torch" control runs with TF32 off, so its unit is float32's.
# Measured on one H100 80GB HBM3 at 700 W (worst |error| / (u max|ref|) for scores, / (u sum|terms|) for gradients):
#   "torch" control, TF32 off: scores 152 u; relative 2-norms up to 9.5e-3; a share of up to 1.95e-2 of the head's
#   second weight gradient past C_GRAD: a flipped ReLU input of that layer moves a whole row of it (1 / 256 of the
#   elements), here about five rows; the kNN module's own max-site margins down to 1.7e-7 relative;
#   "fused" and "fused_all": scores 17.4 u (KITTI coarse head), gradients 12.4 u, no element past C_GRAD; relative
#   2-norms up to 0.29 (first_pointnet).
# REL_GRAD bounds every per-parameter relative 2-norm.  With the arg-maxes aligned, what is left in the fused modes is
# ReLU inputs within TF32 rounding of zero: the scores differ by up to ~1e-2 of max|ref|, a share of that order of the
# ReLU inputs flips, and with a random cotangent each flip moves one whole term of a sum of random-sign terms, so a
# weight gradient moves by about sqrt(share) ~ 0.1 relative, growing with depth (0.03 at the head's last layer, 0.08
# at its second, 0.1-0.29 below).  That is as large as the arg-max flips the 2^-1 of the loose whole-model tests was
# set for, so the fused modes keep 2^-1 there; the per-element bounds, the scores and the running statistics are what
# is tight.  At float32 the flips are ~2^13 times rarer, and the control holds 2^-5.
BOUNDS = {"torch": (2.0 ** -24, 256, 256, 2.0 ** -5, 2.0 ** -5),
          "fused": (2.0 ** -10, 32, 16, 1e-2, 2.0 ** -1),
          "fused_all": (2.0 ** -10, 32, 16, 1e-2, 2.0 ** -1)}

# name -> (img_H, img_W, fine, B, N, Ma, Mb, k_ab)
SHAPES = {"small": (64, 128, True, 2, 2048, 128, 128, 16),
          "kitti": (160, 512, True, 2, 20480, 128, 128, 16),
          "kitti_coarse": (160, 512, False, 2, 20480, 128, 128, 16),
          "oxford": (384, 640, True, 2, 20480, 128, 128, 16),
          "nodes": (64, 128, True, 2, 4096, 96, 64, 8)}
WRAPPED = ("cluster_assign_forward", "cluster_max_pool", "knn_group", "upsample_by_interpolation",
           "attention_fusion", "channel_product", "point_chain", "point_branch")
SITE = {("pc", "node_a"): "pa", ("pc", "node_b"): "pb", ("node_a", "node_b"): "ab"}


class Recorder:
    """Wraps WRAPPED in point_ops; each call appends (op, bound arguments, result, extra), extra holding what the
    call consumes: a copy of a group-max point_branch's layers and the dropout state as they were before it."""

    def __init__(self, monkeypatch, model):
        self.calls, self.hooked, self.maps = [], {}, {}
        self.real = {name: getattr(point_ops, name) for name in WRAPPED}
        for name in WRAPPED:
            monkeypatch.setattr(point_ops, name, self._wrap(name))
        knn, final = model.pc_encoder.knnlayer, model.pc_encoder.final_pointnet
        self.handles = [knn.layers_before[-1].register_forward_hook(self._max_hook("knn_before", 3)),
                        knn.layers_after[-1].register_forward_hook(self._max_hook("knn_after", 3)),
                        final.register_forward_hook(self._max_hook("global", 2)),
                        model.img_encoder.backbone.register_forward_hook(self._maps)]

    def _wrap(self, name):
        real, sig = self.real[name], inspect.signature(self.real[name])

        def op(*args, **kwargs):
            a = sig.bind(*args, **kwargs)
            a.apply_defaults()
            a = dict(a.arguments)
            extra = {}
            if name in ("point_chain", "point_branch"):
                if isinstance(a.get("drop_state"), torch.Tensor):
                    extra["drop_state"] = a["drop_state"].clone()
                if a.get("max_group") is not None:
                    extra["layers"] = copy.deepcopy(list(a["layers"]))
            if name == "cluster_max_pool":
                extra["features"] = a["features"].detach().clone()
            out = real(*args, **kwargs)
            self.calls.append((name, a, out, extra))
            return out
        return op

    def _max_hook(self, site, dim):
        def hook(mod, inp, out):
            self.hooked[site] = first_argmax(out.detach(), dim)
        return hook

    def _maps(self, mod, inp, out):
        """The image maps as leaves, so the gradients reaching them are the image branch's incoming ones."""
        self.maps = {k: t.detach().requires_grad_() for k, t in zip(("s16", "s32"), out)}
        return self.maps["s16"], self.maps["s32"]

    def close(self):
        for h in self.handles:
            h.remove()


def _which(t, x):
    for k in ("pc", "node_a", "node_b"):
        if tuple(t.shape) == tuple(x[k].shape) and torch.equal(t, x[k]):
            return k
    raise AssertionError("a search on coordinates that are not an input")


def _img_global_hook(scores, s32, store):
    """Registers a hook on the mean over s32's pixels (the global image feature): store["img_global"] receives its
    incoming gradient.  There must be exactly one such node in the graph."""
    seen, found, stack = set(), [], [scores.grad_fn]
    while stack:
        node = stack.pop()
        if node is None or node in seen:
            continue
        seen.add(node)
        nxt = [f for f, _ in node.next_functions]
        if "Mean" in node.name() and any(getattr(f, "variable", None) is s32 for f in nxt if f is not None):
            found.append(node)
        stack += nxt
    assert len(found) == 1, f"{len(found)} means over the stride-32 map in the graph"

    def hook(grad_inputs, grad_outputs):
        store["img_global"] = grad_outputs[0]
    found[0].register_hook(hook)


def decisions(rec, model, x):
    """The decisions the recorded run made, by DECISIONS name, and the head's dropout masks."""
    dec, keep = {}, None
    knn, final = model.pc_encoder.knnlayer, model.pc_encoder.final_pointnet
    branch_site = {id(knn.layers_before[0]): "knn_before", id(knn.layers_after[0]): "knn_after",
                   id(final.layers[0]): "global"}

    def put(site, idx):
        assert site not in dec or torch.equal(dec[site], idx), f"two calls disagree on {site}"
        dec[site] = idx

    assign = [(SITE[_which(a["pc"], x), _which(a["node"], x)], out["min_k_idx"].long())
              for name, a, out, _ in rec.calls if name == "cluster_assign_forward"]
    for name, a, out, extra in rec.calls:
        if name == "upsample_by_interpolation":
            put(SITE[_which(a["query"], x), _which(a["node"], x)], a["topk_idx"].long())
        elif name == "knn_group":
            put("knn", out[0].long())
        elif name == "cluster_max_pool":
            f = extra["features"]
            site = {32: "cluster_first", 64: "cluster_second"}[f.shape[1]]
            put(site, point_ops.index_max_forward(f.contiguous(), a["min_idx"], a["M"]).long())
        elif name == "point_branch" and a["max_group"] is not None:
            site, G = branch_site[id(a["layers"][0])], a["max_group"]
            state = extra.get("drop_state")
            with torch.no_grad():
                act, mx = rec.real["point_branch"]([s.detach() for s in a["sources"]], extra["layers"], state,
                                                   a["cols"], None if a["add"] is None else a["add"].detach(),
                                                   a["add_group"], G, "both")
            B, C, n = act.shape
            idx = first_argmax(act.reshape(B, C, n // G, G), 3)
            rec_max = out[1] if isinstance(out, tuple) else out
            assert torch.equal(act.reshape(B, C, n // G, G).gather(3, idx).squeeze(3), rec_max), \
                f"{site}: the rerun's group max is not the recorded one"
            put(site, idx if site != "global" else idx.reshape(B, C, 1))
        elif name == "point_chain" and a["layers"][0] is model.per_point_pn.layers[0]:
            N = a["sources"][0].shape[2]
            B = a["sources"][0].shape[0]
            for i, layer in enumerate(a["layers"]):
                if layer.dropout is not None:
                    keep = keep or {}
                    keep[f"per_point_pn.layers.{i}"] = point_ops.point_chain_dropout_mask(
                        extra["drop_state"], i, layer.dropout.p, B, layer.conv.out_channels, N)
    for site, idx in rec.hooked.items():
        put(site, idx)
    for site, idx in assign:            # a search with fewer neighbours than the interpolation's gives its first ones
        if site in dec:
            assert torch.equal(dec[site][..., :idx.shape[2]], idx), f"two calls disagree on {site}"
        else:
            put(site, idx)
    if "pa" in dec:
        for name, a, out, extra in rec.calls:
            if name == "cluster_max_pool":
                assert torch.equal(a["min_idx"].long(), dec["pa"][:, :, 0]), "pooled over another assignment"
    return dec, keep


def _measure(got, want, scale, u, c, frac, what):
    """Per element |got - want| <= c u scale for all but a share frac; prints the worst ratio and the share."""
    err = (got.double() - want.double()).abs()
    ratio = err / (u * scale.double()).clamp_min(1e-300)
    share = (ratio > c).double().mean().item()
    print(f"  {what}: worst {ratio.max().item():.2e} u, share past {c} u {share:.2e}")
    assert share <= frac, f"{what}: {share:.2e} of the elements exceed {c} u (allowed {frac})"
    return ratio.max().item(), share


def _out(got, want, u, c, what):
    scale = want.double().abs().max()
    return _measure(got, want, torch.full_like(want.double(), scale.item()), u, c, 0.0, what)


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-300)).item()


def _normed_bias(model, k):
    return k.endswith("conv.bias") and model.get_submodule(k[:-len(".conv.bias")]).norm is not None


# Gradients that are zero plus rounding on both sides, so no relative 2-norm is taken of them (their per-element check
# against sum|terms| still holds): a conv bias followed by batch-statistics BatchNorm, and these three, each a sum over
# the whole batch of a gradient that reaches the loss only through batch-statistics BatchNorm (via weights that sum to
# one: a broadcast over the nodes, the interpolations), whose input gradient sums to zero over the batch.
BATCH_CANCELLING = {"pc_encoder.final_pointnet.layers.1.norm.bias", "node_b_pn.layers.2.conv.bias",
                    "node_a_pn.layers.2.conv.bias"}


def _run(monkeypatch, mode, shape, dropout, seed=0):
    H, W, fine, B, N, Ma, Mb, k_ab = SHAPES[shape]
    L = network.classifier.fine_grid(H, W, 32)
    L = L[0] * L[1]
    model = network.KeypointDetector(img_H=H, img_W=W, fine=fine, node_a_num=Ma, node_b_num=Mb, k_ab=k_ab,
                                      point_layers=mode)
    model.load_state_dict(synthetic.seeded_state_dict(model, 100 + seed))
    model = model.cuda().train()
    if dropout:
        model.point_chain_state.copy_(point_ops.new_dropout_state(11 + seed, "cuda"))
    else:
        for layer in model.per_point_pn.layers:
            layer.dropout = None
    inp = synthetic.make_network_inputs(20 + seed, B, N, Ma, Mb, H, W, L)
    x = {k: torch.from_numpy(v).cuda() for k, v in inp.items() if k not in ("lw_coarse", "lw_fine")}
    before = state64(model)
    tracked = {k: v.clone() for k, v in model.state_dict().items() if k.endswith("num_batches_tracked")}

    rec = Recorder(monkeypatch, model)
    out = model(x["pc"], x["intensity"], x["sn"], x["node_a"], x["node_b"], x["img"])
    scores = torch.cat(out, dim=1) if fine else out
    store = {}
    s16, s32 = rec.maps["s16"], rec.maps["s32"]
    _img_global_hook(scores, s32, store)
    cot = torch.randn(scores.shape, device="cuda", generator=torch.Generator(device="cuda").manual_seed(5 + seed))
    scores.backward(cot)
    rec.close()
    dec, keep = decisions(rec, model, x)
    assert (keep is not None) == dropout
    print(f"{mode} {shape} dropout {'on' if dropout else 'off'}: ops {sorted({c[0] for c in rec.calls})}, "
          f"decisions recorded {sorted(dec)}")

    # the twin, along the recorded decisions ("torch": the maxes over K and the nodes are decided by the twin itself,
    # and must come out as torch.max's)
    own = {"knn_before", "knn_after", "global"} if mode == "torch" else set()
    given = {k: v for k, v in dec.items() if k not in own}
    assert set(given) | own == set(DECISIONS), f"decisions missing: {set(DECISIONS) - set(given) - own}"
    x64 = {k: v.double() for k, v in x.items()}
    maps = {k: v.detach().double().requires_grad_() for k, v in (("s16", s16), ("s32", s32))}
    maps["ig"] = maps["s32"].detach().mean(dim=(2, 3)).requires_grad_()
    kw = dict(momentum=0.1, k_ab=k_ab, k_interp=3)
    t = Twin(before, dec=given, keep=keep, **kw)
    ref = t.scores(x64["pc"], x64["intensity"], x64["sn"], x64["node_a"], x64["node_b"], maps["s16"], maps["s32"],
                   maps["ig"])
    ref.backward(cot.double())
    for site in own:                    # a group whose maximum is a ReLU zero passes no gradient whatever it picks
        live = t.maxima[site] > 0
        assert torch.equal(t.dec[site][live], dec[site][live]), f"{site}: the twin's own arg-max is not torch.max's"
    if own:
        print("  the twin's own max-site margins:", {k: f"{t.margins[k]:.2e}" for k in sorted(own)})
    mag_P = {k: v.detach().abs().requires_grad_(v.requires_grad) for k, v in before.items()}
    mag_maps = {k: v.detach().abs().requires_grad_() for k, v in maps.items()}
    ta = Twin(mag_P, mag=t, keep=keep, **kw)
    ref_a = ta.scores(x64["pc"], x64["intensity"].abs(), x64["sn"].abs(), x64["node_a"], x64["node_b"],
                      mag_maps["s16"], mag_maps["s32"], mag_maps["ig"])
    ref_a.backward(cot.double().abs())

    u, c_out, c_grad, frac, rel_grad = BOUNDS[mode]
    worst = {"out": 0.0, "grad": 0.0, "share": 0.0}

    def note(kind, r):
        worst[kind] = max(worst[kind], r[0])
        if kind == "grad":
            worst["share"] = max(worst["share"], r[1])
    note("out", _out(scores.detach(), ref.detach(), u, c_out, "scores"))
    params = dict(model.named_parameters())
    rels = {}
    for k, p in before.items():
        if not p.requires_grad:
            continue
        got = params[k].grad
        assert got is not None, f"{k}: no gradient"
        note("grad", _measure(got.reshape(p.shape), p.grad, mag_P[k].grad, u, c_grad, frac, f"grad {k}"))
        if not _normed_bias(model, k) and k not in BATCH_CANCELLING:
            rels[k] = _rel(got.reshape(p.shape), p.grad)
    hw = s32.shape[2] * s32.shape[3]
    s32_want = maps["s32"].grad + maps["ig"].grad[:, :, None, None] / hw
    s32_mag = mag_maps["s32"].grad + mag_maps["ig"].grad[:, :, None, None] / hw
    for what, got, want, mag in (("s16", s16.grad, maps["s16"].grad, mag_maps["s16"].grad),
                                 ("s32", s32.grad, s32_want, s32_mag),
                                 ("img_global", store["img_global"], maps["ig"].grad, mag_maps["ig"].grad)):
        note("grad", _measure(got, want, mag, u, c_grad, frac, f"grad at {what}"))
        rels[what] = _rel(got, want)
    state = model.state_dict()
    for k, v in t.running.items():
        note("out", _out(state[k], v, u, c_out, k))
    for k, v in tracked.items():
        if not k.startswith("img_encoder."):
            assert state[k].item() == v.item() + 1, k
    bad = {k: v for k, v in rels.items() if v >= rel_grad}
    top = max(rels, key=rels.get)
    print(f"  worst: outputs {worst['out']:.2e} u, gradients {worst['grad']:.2e} u, share past {c_grad} u "
          f"{worst['share']:.2e}, relative 2-norm {rels[top]:.2e} ({top})")
    assert not bad, f"relative 2-norms at or above {rel_grad}: {bad}"


@pytest.fixture
def tf32_off():
    flags = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = flags


@pytest.mark.parametrize("shape", ["small", "kitti"])
def test_torch_layers_control_at_float32(monkeypatch, tf32_off, shape):
    """The twin and the recorder on the torch layers with TF32 off: float32-level agreement validates both before they
    judge the fused modes."""
    _run(monkeypatch, "torch", shape, False)


@pytest.mark.parametrize("dropout", [False, True], ids=["dropout_off", "dropout_on"])
@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("mode", ["fused", "fused_all"])
def test_fused_training_matches_the_twin(monkeypatch, mode, shape, dropout):
    _run(monkeypatch, mode, shape, dropout)
