"""The classifier network's construction on the CPU (DESIGN.md 4.18): the state_dict keys and shapes of the reference's
KeypointDetector at the three shipped sizes and both heads, checkpoint loading, the configuration checks, and that
constructing the model touches neither CUDA nor the network."""
import os
import socket

import numpy as np
import pytest
import torch

from deepi2p_b200 import network, synthetic

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "network_small.npz")


@pytest.fixture(scope="module")
def golden():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


@pytest.fixture
def no_cuda_no_network(monkeypatch):
    """Any CUDA initialisation or socket connection raises."""
    def refuse(*args, **kwargs):
        raise AssertionError("touched CUDA or the network")
    monkeypatch.setattr(torch.cuda, "_lazy_init", refuse)
    monkeypatch.setattr(socket.socket, "connect", refuse)
    monkeypatch.setattr(socket, "create_connection", refuse)


def key_list(model):
    return [k + ":" + ",".join(str(d) for d in v.shape) for k, v in model.state_dict().items()]


@pytest.mark.parametrize("shape", ["kitti", "oxford", "nuscenes"])
@pytest.mark.parametrize("fine", [True, False])
def test_state_dict_matches_reference(golden, shape, fine, no_cuda_no_network):
    model = network.KeypointDetector(**network.SHAPES[shape], fine=fine)
    assert key_list(model) == list(golden[f"keys_{shape}_{'fine' if fine else 'coarse'}"])
    assert all(v.device.type == "cpu" for v in model.state_dict().values())


def small_model(**kw):
    return network.KeypointDetector(img_H=64, img_W=128, **kw)


def test_load_checkpoint_prefix_and_errors(tmp_path):
    model = small_model()
    sd = synthetic.seeded_state_dict(model, 3)
    path = tmp_path / "ckpt.pth"
    torch.save({"module." + k: v for k, v in sd.items()}, path)        # DataParallel's layout
    network.load_checkpoint(model, str(path))
    for k, v in model.state_dict().items():
        assert torch.equal(v, sd[k]), k
    other = small_model()
    network.load_checkpoint(other, sd)                                  # plain dict, no prefix
    assert torch.equal(other.per_point_pn.layers[2].conv.weight, sd["per_point_pn.layers.2.conv.weight"])

    missing = dict(sd)
    del missing["node_a_pn.layers.0.norm.running_var"]
    with pytest.raises(KeyError, match=r"node_a_pn\.layers\.0\.norm\.running_var"):
        network.load_checkpoint(small_model(), missing)
    extra = dict(sd, **{"pc_encoder.extra.weight": torch.zeros(1)})
    with pytest.raises(KeyError, match=r"pc_encoder\.extra\.weight"):
        network.load_checkpoint(small_model(), extra)
    with pytest.raises(KeyError, match="node_b_pn"):
        network.load_checkpoint(small_model(), {"module." + k: v for k, v in sd.items() if "node_b_pn" not in k})
    wrong = dict(sd, **{"per_point_pn.layers.2.conv.bias": torch.zeros(3)})
    with pytest.raises(RuntimeError, match="size mismatch"):
        network.load_checkpoint(small_model(), wrong)


def test_configuration_errors_before_cuda(no_cuda_no_network):
    with pytest.raises(ValueError, match="normalization"):
        network.KeypointDetector(normalization="instance")
    with pytest.raises(ValueError, match="activation"):
        network.KeypointDetector(activation="elu")
    # 100 x 512: the stride-32 map is 4 x 16, the fine grid round(100 / 32) x 16 = 3 x 16
    with pytest.raises(ValueError, match="stride-32"):
        network.KeypointDetector(img_H=100, img_W=512)
    with pytest.raises(ValueError, match="stride-32"):
        network.KeypointDetector(img_H=160, img_W=512, fine_scale=16)


def test_construct_offline_and_resnet_file(tmp_path, no_cuda_no_network):
    model = network.KeypointDetector(**network.SHAPES["oxford"])
    assert all(p.device.type == "cpu" for p in model.parameters())
    backbone = synthetic.seeded_state_dict(model.img_encoder.backbone, 5)
    path = tmp_path / "resnet34.pth"
    torch.save(backbone, path)
    loaded = network.KeypointDetector(**network.SHAPES["kitti"], resnet_weights=path)
    for k, v in loaded.img_encoder.backbone.state_dict().items():
        assert torch.equal(v, backbone[k]), k
    assert "fc.weight" in backbone and "layer4.2.bn2.running_var" in backbone       # torchvision's layout


def test_initialisation_rule():
    torch.manual_seed(0)
    model = network.KeypointDetector(img_H=64, img_W=128)
    conv = model.node_b_pn.layers[0].conv                               # 1792 -> 1024, N(0, sqrt(2 / 1792))
    assert abs(float(conv.weight.detach().std()) - (2.0 / 1792) ** 0.5) < 0.02 * (2.0 / 1792) ** 0.5
    assert float(conv.bias.detach().abs().max()) == 0.0
    bn = model.node_b_pn.layers[0].norm
    assert torch.equal(bn.weight, torch.ones_like(bn.weight)) and torch.equal(bn.bias, torch.zeros_like(bn.bias))
    rconv = model.img_encoder.backbone.layer4[0].conv1                  # kaiming fan_out: sqrt(2 / (512 * 9))
    assert abs(float(rconv.weight.detach().std()) - (2.0 / (512 * 9)) ** 0.5) < 0.02 * (2.0 / (512 * 9)) ** 0.5
    assert [type(m).__name__ for m in model.per_point_pn.layers[0].modules()].count("Dropout") == 1
    assert model.per_point_pn.layers[2].dropout is None and model.per_point_pn.layers[2].norm is None


def test_seeded_state_dict_is_reproducible():
    model = small_model(fine=False)
    a, b = synthetic.seeded_state_dict(model, 11), synthetic.seeded_state_dict(model, 11)
    assert list(a) == sorted(model.state_dict())
    assert all(torch.equal(a[k], b[k]) for k in a)
    assert all(float(v.min()) >= 0.5 for k, v in a.items() if k.endswith("running_var"))
    assert a["pc_encoder.first_pointnet.layers.0.norm.num_batches_tracked"].dtype == torch.int64


def test_predict_rule():
    coarse = torch.tensor([[[1.0, 2.0, 3.0, float("nan")], [1.0, 1.0, 4.0, 0.0]]])
    fine = torch.tensor([[[0.0, 5.0], [2.0, 5.0], [2.0, float("nan")]]])
    c, f = network.predict(coarse, fine)
    assert c.dtype == torch.int8 and f.dtype == torch.int32
    assert c.tolist() == [[0, 0, 1, 0]]                     # ties -> first index, NaN is maximal
    assert f.tolist() == [[1, 2]]
    assert network.predict(coarse)[1] is None


def test_fixture_inputs_regenerate(golden):
    """The reference fixture stores no inputs: its seed regenerates them, and the stored sums pin the generator."""
    x = synthetic.make_network_inputs(int(golden["input_seed"]))
    assert sorted(x) == list(golden["input_names"])
    sums = [x[k].astype(np.float64).sum() for k in golden["input_names"]]
    assert np.array_equal(np.array(sums), golden["input_sums"])
    assert x["pc"].shape == (2, 3, 2048) and x["img"].shape == (2, 3, 64, 128) and x["lw_fine"].shape == (2, 8, 2048)


def test_forward_needs_cuda():
    model = small_model().eval()
    B, N = 1, 256
    args = (torch.zeros(B, 3, N), torch.zeros(B, 1, N), torch.zeros(B, 3, N), torch.rand(B, 3, 128),
            torch.rand(B, 3, 128), torch.zeros(B, 3, 64, 128))
    with pytest.raises(RuntimeError, match="CUDA"):
        model(*args)
