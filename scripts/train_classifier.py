"""Train the classifier from a KITTI, Oxford or nuScenes root: {kitti,oxford,nuscenes_t}/train_classifier.py on the
GPU, with the reference's schedule, test pass, loss lines and checkpoint names (deepi2p_b200.train, DESIGN.md 4.32).

    python scripts/train_classifier.py --dataset {kitti,oxford,nuscenes} --root R --out DIR
        [--epochs 101] [--batch B] [--seed 0] [--version V] [--coarse-only] [--resnet-weights FILE]
        [--record-dir NAME] [--nuscenes-version V] [--resume DIR/resume.pth] [--store {cuda,pinned}]
        [--point-layers {torch,fused,fused_all}] [--precision {fp32,bf16}]

Every epoch writes DIR/v{version}-gpu{gpu}-epoch{epoch}-{test coarse accuracy}.pth (the detector's state_dict, which
network.load_checkpoint and the reference's load_model read) and DIR/resume.pth (model, optimiser, epoch, step
count, lr and seed), from which --resume continues.
"""
import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from deepi2p_b200 import network, train  # noqa: E402


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description="train the DeepI2P classifier")
    ap.add_argument("--dataset", required=True, choices=train.DATASETS)
    ap.add_argument("--root", required=True)
    ap.add_argument("--out", required=True, help="folder of the checkpoints and resume.pth")
    ap.add_argument("--epochs", type=int, default=train.EPOCHS)
    ap.add_argument("--batch", type=int, default=None, help="batch size (default: the dataset's options.py value)")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--version", default=None, help="checkpoint name version (default: the dataset's options.py)")
    ap.add_argument("--coarse-only", action="store_true", help="MMClassiferCoarse: no fine head, coarse alpha 1")
    ap.add_argument("--resnet-weights", default=None, help="local torchvision ResNet-34 state_dict to start from")
    ap.add_argument("--record-dir", default=None, help="KITTI scan record folder (default voxel0.1-SNr0.6)")
    ap.add_argument("--nuscenes-version", default=None,
                    help="nuScenes table version of both splits (default v1.0-trainval / v1.0-test)")
    ap.add_argument("--resume", default=None, help="a resume.pth to continue from")
    ap.add_argument("--store", default=None, choices=("cuda", "pinned"),
                    help="keep the scan records in one device or pinned store (KITTI, Oxford)")
    ap.add_argument("--point-layers", default="torch", choices=network.POINT_LAYERS,
                    help="fused: the per-point chains as point_ops.point_chain (TF32, its own dropout stream); "
                         "fused_all: also the kNN module, final_pointnet and the node-level PointNets as "
                         "point_ops.point_branch")
    ap.add_argument("--precision", default="fp32", choices=train.PRECISIONS,
                    help="bf16: the forward and the loss under bfloat16 autocast (with --point-layers torch only); "
                         "parameters, optimiser state and checkpoints stay float32")
    a = ap.parse_args(argv)
    if a.epochs < 1:
        ap.error("--epochs must be >= 1")
    if a.batch is not None and a.batch < 1:
        ap.error("--batch must be >= 1")
    if a.record_dir is not None and a.dataset != "kitti":
        ap.error("--record-dir is a KITTI setting")
    if a.nuscenes_version is not None and a.dataset != "nuscenes":
        ap.error("--nuscenes-version is a nuScenes setting")
    if a.store is not None and a.dataset == "nuscenes":
        ap.error("--store: nuScenes batches read their sweeps from the files")
    if a.precision == "bf16" and a.point_layers != "torch":
        ap.error("--precision bf16 needs --point-layers torch")
    return a


def main(argv=None):
    a = parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("train_classifier.py needs a CUDA device")
    model = network.KeypointDetector(**network.SHAPES[a.dataset], fine=not a.coarse_only,
                                     resnet_weights=a.resnet_weights, point_layers=a.point_layers).cuda()
    src = lambda mode: train.batch_source(a.dataset, a.root, mode, store=a.store, record_dir=a.record_dir,
                                          nuscenes_version=a.nuscenes_version)
    trainset, testset = src("train"), src("val")
    print("#training point clouds = %d" % trainset[0])
    print("#testing point clouds = %d" % testset[0])
    trainer = train.Trainer(model, trainset, testset, a.dataset, a.out, batch_size=a.batch, seed=a.seed,
                            epochs=a.epochs, version=a.version, precision=a.precision)
    if a.resume:
        trainer.resume(a.resume)
    return trainer.run()


if __name__ == "__main__":
    main()
