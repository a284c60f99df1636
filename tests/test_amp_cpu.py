"""bfloat16 autocast without a GPU (DESIGN.md 4.37): the ops' dtype rules (bf16 feature operands pass, a mix of
float32 and bf16 and any other dtype raise with the stated messages), the header's bf16 entry points, the network's and
the trainer's raises, and train_classifier.py's --precision."""
import os
import sys

import pytest
import torch

from deepi2p_b200 import _native, build, classifier, network, point_ops, train

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BF = torch.bfloat16


def _past_dtype_checks(fn, *args):
    """The checks run in order, dtype and shape first, device last: a CPU call that gets as far as the device check
    passed every dtype check."""
    with pytest.raises(RuntimeError, match="must be a CUDA tensor"):
        fn(*args)


def test_bf16_operands_pass_the_dtype_checks():
    f = torch.zeros(2, 4, 10, dtype=BF)
    idx = torch.zeros(2, 10, dtype=torch.int32)
    _past_dtype_checks(point_ops.cluster_max_pool, f, idx, 3)
    _past_dtype_checks(point_ops.knn_group, torch.zeros(2, 3, 5), torch.zeros(2, 3, 10), f, 4)
    _past_dtype_checks(point_ops.upsample_by_interpolation, torch.zeros(2, 7, 3, dtype=torch.int32),
                       torch.zeros(2, 3, 7), torch.zeros(2, 3, 10), f)
    _past_dtype_checks(point_ops.attention_fusion, f, torch.zeros(2, 10, 6, dtype=BF))
    _past_dtype_checks(classifier.classifier_loss, torch.zeros(2, 2, 10, dtype=BF), torch.zeros(2, 80, 10, dtype=BF),
                       torch.zeros(2, 3, 10), torch.zeros(2, 3, 4), torch.zeros(2, 3, 3), 160, 512)
    _past_dtype_checks(classifier.classifier_loss, torch.zeros(2, 2, 10, dtype=BF), None, torch.zeros(2, 3, 10),
                       torch.zeros(2, 3, 4), torch.zeros(2, 3, 3), 160, 512)


def test_mixed_feature_dtypes_raise_naming_both():
    with pytest.raises(RuntimeError, match="img_features and attention must have the same dtype"):
        point_ops.attention_fusion(torch.zeros(2, 4, 10, dtype=BF), torch.zeros(2, 10, 6))
    with pytest.raises(RuntimeError, match="img_features and attention must have the same dtype"):
        point_ops.attention_fusion(torch.zeros(2, 4, 10), torch.zeros(2, 10, 6, dtype=BF))
    with pytest.raises(RuntimeError, match="coarse_scores and fine_scores must have the same dtype"):
        classifier.classifier_loss(torch.zeros(2, 2, 10, dtype=BF), torch.zeros(2, 80, 10), torch.zeros(2, 3, 10),
                                   torch.zeros(2, 3, 4), torch.zeros(2, 3, 3), 160, 512)


@pytest.mark.parametrize("dtype", [torch.float16, torch.float64])
def test_float16_and_float64_features_raise(dtype):
    f = torch.zeros(2, 4, 10, dtype=dtype)
    with pytest.raises(RuntimeError, match="features must have dtype"):
        point_ops.cluster_max_pool(f, torch.zeros(2, 10, dtype=torch.int32), 3)
    with pytest.raises(RuntimeError, match="features must have dtype"):
        point_ops.knn_group(torch.zeros(2, 3, 5), torch.zeros(2, 3, 10), f, 4)
    with pytest.raises(RuntimeError, match="features must have dtype"):
        point_ops.upsample_by_interpolation(torch.zeros(2, 7, 3, dtype=torch.int32), torch.zeros(2, 3, 7),
                                            torch.zeros(2, 3, 10), f)
    with pytest.raises(RuntimeError, match="attention must have dtype"):
        point_ops.attention_fusion(torch.zeros(2, 4, 10, dtype=BF), torch.zeros(2, 10, 6, dtype=dtype))
    with pytest.raises(RuntimeError, match="coarse_scores must have dtype"):
        classifier.classifier_loss(torch.zeros(2, 2, 10, dtype=dtype), None, torch.zeros(2, 3, 10),
                                   torch.zeros(2, 3, 4), torch.zeros(2, 3, 3), 160, 512)
    # the coordinates stay float32 only
    with pytest.raises(RuntimeError, match="query must have dtype"):
        point_ops.knn_group(torch.zeros(2, 3, 5, dtype=BF), torch.zeros(2, 3, 10), torch.zeros(2, 4, 10), 4)


def test_header_declares_a_bf16_twin_of_each_f32_entry_point():
    sigs = _native.parse_header(open(build.HEADER).read())
    for name in ("cluster_pool_forward", "cluster_pool_backward", "knn_group_forward", "knn_group_backward",
                 "interp_forward", "interp_backward", "attn_fusion_forward", "attn_fusion_backward",
                 "classifier_loss_forward", "classifier_loss_backward"):
        assert sigs[name + "_bf16"] == sigs[name + "_f32"], name


def test_network_rejects_autocast_with_fused_layers_and_float16():
    # torch.autocast("cuda") sets the autocast dtype even where CUDA is missing (it warns and disables itself)
    with pytest.warns(UserWarning), torch.autocast("cuda", dtype=BF):
        network.check_autocast("torch")
        for mode in ("fused", "fused_all"):
            with pytest.raises(ValueError, match="point_layers='torch'"):
                network.check_autocast(mode)
    with pytest.warns(UserWarning), torch.autocast("cuda", dtype=torch.float16):
        with pytest.raises(ValueError, match="bfloat16 only"):
            network.check_autocast("torch")


def test_trainer_rejects_bf16_with_fused_layers():
    for mode in ("fused", "fused_all"):
        model = network.KeypointDetector(**network.SHAPES["kitti"], point_layers=mode)
        with pytest.raises(ValueError, match="needs point_layers='torch'"):
            train.Trainer(model, (16, None), (16, None), "kitti", "unused", precision="bf16")
    model = network.KeypointDetector(**network.SHAPES["kitti"])
    with pytest.raises(ValueError, match="precision must be one of"):
        train.Trainer(model, (16, None), (16, None), "kitti", "unused", precision="fp16")
    with pytest.raises(ValueError, match="precision must be one of"):
        train.autocast("fp16")


def test_precision_option_parses():
    sys.path.insert(0, os.path.join(ROOT, "scripts"))
    import train_classifier
    base = ["--dataset", "kitti", "--root", "r", "--out", "o"]
    assert train_classifier.parse_args(base).precision == "fp32"
    assert train_classifier.parse_args(base + ["--precision", "bf16"]).precision == "bf16"
    with pytest.raises(SystemExit):
        train_classifier.parse_args(base + ["--precision", "fp16"])
    with pytest.raises(SystemExit):
        train_classifier.parse_args(base + ["--precision", "bf16", "--point-layers", "fused"])
