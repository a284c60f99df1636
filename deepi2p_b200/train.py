"""Training of the classifier from a dataset root: {kitti,oxford,nuscenes_t}/train_classifier.py with
MMClassifer.optimize / test_model / update_learning_rate / save_network (models/multimodal_classifier.py), on the
project's batch assembly (kitti.kitti_batch, oxford.oxford_batch, nuscenes.nuscenes_batch), network.KeypointDetector
and classifier.classifier_loss (DESIGN.md 4.32).

    model = network.KeypointDetector(**network.SHAPES["kitti"])
    trainer = train.Trainer(model.cuda(), train.batch_source("kitti", root, "train"),
                            train.batch_source("kitti", root, "val"), "kitti", out_dir)
    trainer.run()

One epoch: the train list in a permutation seeded by (seed, epoch), drop_last batches; per batch the step of
MMClassifer.optimize (train mode, forward, classifier_loss, zero_grad, backward, Adam), captured once as a CUDA graph
and replayed; then the test pass over the whole "val" list in order, means weighted by the batch size; then the lr
rule; then the epoch's checkpoint and the resume file.  While step k runs, batch k + 1 is assembled on a side stream,
so the assembly's host reads wait on that stream only.  Losses and accuracies are summed on the device and read at
the print interval and at the end of the epoch: the loop itself never synchronises with the device.
"""
import contextlib
import os
import time

import numpy as np
import torch

from . import classifier, kitti, network, nuscenes, oxford, point_ops

DATASETS = ("kitti", "oxford", "nuscenes")

# per-dataset settings: batch_size and lr_decay_step from {kitti,oxford,nuscenes_t}/options.py (kitti :47 / :54,
# oxford :46 / :53, nuscenes_t :45 / :52), the print interval from each train_classifier.py's `i % int(...)`
# (kitti :70 800, oxford :70 600, nuscenes_t :70 1200), version from each options.py :11
DEFAULTS = {"kitti": dict(batch_size=8, lr_decay_step=20, print_interval=800, version="1.27"),
            "oxford": dict(batch_size=8, lr_decay_step=10, print_interval=600, version="0.1-fine"),
            "nuscenes": dict(batch_size=12, lr_decay_step=15, print_interval=1200, version="3.3")}
LR = 0.001                  # options.py lr (kitti :53, oxford :52, nuscenes_t :51)
BETAS = (0.9, 0.999)        # multimodal_classifier.py:45-48 Adam(betas=(0.9, 0.999), weight_decay=0)
WEIGHT_DECAY = 0.0
LR_DECAY_SCALE = 0.5        # options.py lr_decay_scale (kitti :55, oxford :54, nuscenes_t :53)
LR_CLIP = 0.00001           # multimodal_classifier.py:268 update_learning_rate's lr_clip
EPOCHS = 101                # train_classifier.py: for epoch in range(101)
INPUT_FIELDS = ("pc", "intensity", "sn", "node_a", "node_b", "P", "img", "K")
LOSS_KEYS = ("loss", "coarse", "fine")
ACCURACY_KEYS = ("coarse_accuracy", "fine_accuracy")
WARMUP_STEPS = 3            # eager steps before the capture: Adam's state and every lazy initialisation exist by then
# Trainer(precision=...): "fp32" is the reference's float32 step; "bf16" runs the forward and the loss under bfloat16
# autocast (DESIGN.md 4.37)
PRECISIONS = ("fp32", "bf16")


def coarse_loss_alpha(fine):
    """options.py: coarse_loss_alpha is 50 for the fine classifier and 1 for the coarse-only one (kitti :57-60)."""
    return 50.0 if fine else 1.0


def decayed_lr(lr, epoch, lr_decay_step, scale=LR_DECAY_SCALE, clip=LR_CLIP):
    """The lr after epoch `epoch`'s test pass: update_learning_rate(scale) when epoch % lr_decay_step == 0 and
    epoch > 0 (lr * scale, clipped at 1e-5 from below), else lr unchanged."""
    if epoch % lr_decay_step == 0 and epoch > 0:
        return max(lr * scale, clip)
    return lr


def lr_schedule(epochs, lr_decay_step, lr=LR, scale=LR_DECAY_SCALE, clip=LR_CLIP):
    """The lr each of `epochs` epochs trains with."""
    out = []
    for e in range(epochs):
        out.append(lr)
        lr = decayed_lr(lr, e, lr_decay_step, scale, clip)
    return out


def epoch_order(n, batch_size, seed, epoch):
    """DataLoader(shuffle=True, drop_last=True) restated: a permutation of the n entries from a numpy Generator seeded
    by (seed, epoch), cut into n // batch_size batches; the rest is dropped.  Returns int64 [n // batch_size,
    batch_size]."""
    nb = n // batch_size
    perm = np.random.default_rng([int(seed), int(epoch)]).permutation(n)
    return perm[:nb * batch_size].reshape(nb, batch_size)


def test_batches(n, batch_size):
    """DataLoader(shuffle=False) restated: the entries in order, the last partial batch kept."""
    return [list(range(a, min(a + batch_size, n))) for a in range(0, n, batch_size)]


def batch_draws(seed, epoch, index, test=False):
    """(device seed, numpy Generator) of one batch's assembly, both derived from (seed, epoch, train/test, index)."""
    ss = np.random.SeedSequence([int(seed), int(epoch), int(bool(test)), int(index)])
    return int(ss.generate_state(1, np.uint64)[0]), np.random.default_rng(ss)


def checkpoint_name(version, gpu, epoch, coarse_accuracy):
    """save_network's file name in train_classifier.py: v{version}-gpu{gpu}-epoch{epoch}-{coarse accuracy:%f}.pth."""
    return "v%s-gpu%d-epoch%d-%f.pth" % (version, gpu, epoch, coarse_accuracy)


def weighted_means(sums, samples):
    """The test pass's means: sums of B * value over the batches divided by the sample count (train_classifier.py
    :105-130)."""
    return {k: v / samples for k, v in sums.items()}


def format_losses(losses, accuracies, per_sample_time, fine=True):
    """MMClassifer.print_loss_dict's line ('%.4f' values; MMClassiferCoarse prints '%.3f' / '%.2f')."""
    tf, vf = ("%.4f", "%.4f") if fine else ("%.3f", "%.2f")
    out = ("Per sample time: " + tf + " - ") % per_sample_time
    for k, v in list(losses.items()) + list(accuracies.items()):
        out += ("%s: " + vf + ", ") % (k, v)
    return out


def save_resume(path, model, optimizer, epoch, step, lr, seed, extra=None):
    """The resume file: model and optimiser state, the last finished epoch, the step count, the lr of the next epoch,
    the run's seed and the device's RNG state (dropout's draws continue where they stopped), plus `extra`, written to a temporary name and renamed."""
    dev = next(model.parameters()).device
    state = dict(model=model.state_dict(), optimizer=optimizer.state_dict(), epoch=int(epoch), step=int(step),
                 lr=float(lr), seed=int(seed), cuda_rng=torch.cuda.get_rng_state(dev), extra=dict(extra or {}))
    tmp = path + ".partial"
    torch.save(state, tmp)
    os.replace(tmp, path)


def load_resume(path):
    return torch.load(path, map_location="cpu", weights_only=True)


def batch_source(dataset, root, mode, store=None, record_dir=None, nuscenes_version=None, seqs=None):
    """(entry count, fn(items, seed, rng, stream) -> the loader's tuple) of the `mode` list of a dataset root.

    store "cuda" or "pinned" keeps every scan record of the list's KITTI sequences or Oxford traversals in one ragged
    ScanStore (DESIGN.md 4.22); None reads each batch's records from the files.  record_dir: KITTI's record folder
    (kitti.RECORD_DIR by default); seqs: KITTI sequences other than the mode's (0-8 train, 9 and 10 val).  nuScenes reads <root>/trainval (v1.0-trainval) for train and <root>/test
    (v1.0-test) otherwise, as nuScenesLoader does, unless nuscenes_version names the table version of both."""
    if dataset not in DATASETS:
        raise ValueError(f"dataset must be one of {DATASETS} (got {dataset!r})")
    if store not in (None, "cuda", "pinned"):
        raise ValueError(f"store must be None, 'cuda' or 'pinned' (got {store!r})")
    if dataset == "kitti":
        ds = kitti.KittiDataset(root, mode, seqs, record_dir=record_dir or kitti.RECORD_DIR)
        st = None if store is None else kitti.scan_store(root, sorted({e[0] for e in ds.entries}), store,
                                                         record_dir=ds.record_dir)
        return len(ds), lambda items, seed, rng, stream: kitti.kitti_batch(ds, items, mode, seed, rng=rng, store=st,
                                                                           stream=stream)
    if record_dir is not None or seqs is not None:
        raise ValueError("record_dir and seqs are KITTI settings")
    if dataset == "oxford":
        ds = oxford.OxfordDataset(root, mode)
        st = None if store is None else oxford.scan_store(root, list(ds.traversals), store)
        return len(ds), lambda items, seed, rng, stream: oxford.oxford_batch(ds, items, mode, seed, rng=rng,
                                                                             store=st, stream=stream)
    if store is not None:
        raise ValueError("nuScenes batches read their sweeps from the files: there is no scan store")
    sub, version = ("trainval", "v1.0-trainval") if mode == "train" else ("test", "v1.0-test")
    dataroot = os.path.join(root, sub)
    tables = nuscenes.Tables(dataroot, nuscenes_version or version)
    info = nuscenes.load_dataset_info(os.path.join(dataroot, "dataset_info.list"))
    return len(info), lambda items, seed, rng, stream: nuscenes.nuscenes_batch(tables, [info[i] for i in items], mode,
                                                                               seed, rng=rng, stream=stream)


def make_optimizer(model, lr=LR):
    """The reference's Adam (lr, betas (0.9, 0.999), weight decay 0) with the lr in a device tensor and capturable
    state, so that a captured step reads the current lr and an lr change needs no recapture."""
    dev = next(model.parameters()).device
    return torch.optim.Adam(model.parameters(), lr=torch.tensor(float(lr), dtype=torch.float32, device=dev),
                            betas=BETAS, weight_decay=WEIGHT_DECAY, capturable=True)


def autocast(precision):
    """The context the forward and the loss run in: nothing for "fp32"; for "bf16" torch.autocast("cuda",
    dtype=torch.bfloat16) with the weight-cast cache off, so that a captured step casts the weights it reads at replay
    time.  No GradScaler is needed: bfloat16 has float32's exponent range."""
    if precision not in PRECISIONS:
        raise ValueError(f"precision must be one of {PRECISIONS}, got {precision!r}")
    if precision == "fp32":
        return contextlib.nullcontext()
    return torch.autocast("cuda", dtype=torch.bfloat16, cache_enabled=False)


def _forward_loss(model, inputs, precision):
    with autocast(precision):
        scores = model(*(inputs[k] for k in ("pc", "intensity", "sn", "node_a", "node_b", "img")))
        coarse, fine = scores if model.fine else (scores, None)
        return classifier.classifier_loss(coarse, fine, inputs["pc"], inputs["P"], inputs["K"], model.img_H,
                                          model.img_W, model.fine_scale, coarse_loss_alpha=coarse_loss_alpha(model.fine))


def train_step(model, optimizer, inputs, precision="fp32"):
    """MMClassifer.optimize on one batch (INTEGRATION.md 4d): train mode, forward, classifier_loss, zero_grad,
    backward, optimizer step.  inputs: INPUT_FIELDS -> device tensors.  precision "bf16" runs the forward and the loss
    under autocast(precision); the backward and Adam run outside it, on the float32 parameters.  Returns
    classifier_loss's dict."""
    model.train()
    out = _forward_loss(model, inputs, precision)
    optimizer.zero_grad(set_to_none=True)
    out["loss"].backward()
    optimizer.step()
    return out


def _stats(out):
    """[loss, coarse, fine, coarse_accuracy, fine_accuracy] as one device vector (zeros for a coarse-only model)."""
    z = out["coarse"].new_zeros(())
    return torch.stack([out["loss"].detach(), out["coarse"].detach(),
                        z if out["fine"] is None else out["fine"].detach(), out["coarse_accuracy"],
                        z if out["fine_accuracy"] is None else out["fine_accuracy"]])


class Trainer:
    """The training loop of train_classifier.py for a KeypointDetector on the device.

    train_source / test_source: batch_source results.  The step is captured as one CUDA graph after WARMUP_STEPS
    eager steps (forward, loss, backward, Adam, BatchNorm statistics and dropout with torch's graph-safe RNG) and
    replayed from one static input set; the assembled batch goes through a staging buffer filled on a side stream
    while the previous step runs.  Checkpoints and the resume file go to out_dir.  gpu: the number in the checkpoint
    names (the device index by default).  precision: "fp32" (the reference's) or "bf16" (the step and the test pass
    under bfloat16 autocast, point_layers="torch" only; parameters, Adam's state, BatchNorm's buffers and the
    checkpoints stay float32)."""

    def __init__(self, model, train_source, test_source, dataset, out_dir, batch_size=None, seed=0, epochs=EPOCHS,
                 version=None, gpu=None, log=print, precision="fp32"):
        if not isinstance(model, network.KeypointDetector):
            raise TypeError("Trainer trains a network.KeypointDetector")
        if precision not in PRECISIONS:
            raise ValueError(f"precision must be one of {PRECISIONS}, got {precision!r}")
        if precision == "bf16" and model.point_layers != "torch":
            raise ValueError(f"precision='bf16' needs point_layers='torch', the model has {model.point_layers!r}: the "
                             f"fused point layers are float32 TF32 kernels")
        self.precision = precision
        d = DEFAULTS[dataset]
        self.model, self.dataset, self.out_dir, self.log = model, dataset, out_dir, log
        self.batch_size = int(batch_size or d["batch_size"])
        self.lr_decay_step, self.print_interval = d["lr_decay_step"], d["print_interval"]
        self.version = d["version"] if version is None else version
        self.seed, self.epochs = int(seed), int(epochs)
        self.device = next(model.parameters()).device
        self.gpu = self.device.index if gpu is None else int(gpu)
        self.n_train, self.make_train = train_source
        self.n_test, self.make_test = test_source
        if self.n_train < self.batch_size:
            raise ValueError(f"the train list has {self.n_train} entries, fewer than one batch of {self.batch_size}")
        self.optimizer = make_optimizer(model)
        self.lr = LR
        self.epoch, self.step_count, self.best = 0, 0, 0.0
        self.side = torch.cuda.Stream(self.device)
        self.inputs = self.staging = None
        self.graph, self._eager_steps = None, 0
        self.sums = torch.zeros(5, dtype=torch.float64, device=self.device)
        self._consumed = torch.cuda.Event()
        if model.point_layers in ("fused", "fused_all"):   # point_chain's dropout stream starts from the run's seed
            model.point_chain_state.copy_(point_ops.new_dropout_state(self.seed, self.device))

    # -- state --------------------------------------------------------------------------------------------------------
    def _set_lr(self, lr):
        self.lr = float(lr)
        for g in self.optimizer.param_groups:
            g["lr"].fill_(self.lr)

    def resume(self, path):
        """Continue from a resume file: model, optimiser, next epoch, step count, lr and seed."""
        st = load_resume(path)
        self.model.load_state_dict(st["model"])
        lr_t = self.optimizer.param_groups[0]["lr"]
        self.optimizer.load_state_dict(st["optimizer"])
        for g in self.optimizer.param_groups:
            g["lr"] = lr_t
        self._set_lr(st["lr"])
        self.epoch, self.step_count, self.seed = st["epoch"] + 1, st["step"], st["seed"]
        torch.cuda.set_rng_state(st["cuda_rng"], self.device)
        self.best = float(st["extra"].get("best", 0.0))
        if "point_chain_state" in st["extra"]:
            self.model.point_chain_state.copy_(st["extra"]["point_chain_state"])
        self.graph, self._eager_steps = None, 0

    # -- input buffers -------------------------------------------------------------------------------------------------
    def _load(self, items, seed, rng, make):
        """Assemble one batch on the side stream into the staging buffer; returns the event that marks it ready."""
        with torch.cuda.stream(self.side):
            self.side.wait_event(self._consumed)          # the previous batch has left the staging buffer
            t = make(items, seed, rng, self.side)
            vals = dict(zip(INPUT_FIELDS, t[:8]))
            if self.staging is None:
                self.staging = {k: torch.empty(v.shape, dtype=torch.float32, device=self.device)
                                for k, v in vals.items()}
            for k, v in vals.items():
                self.staging[k].copy_(v.to(torch.float32), non_blocking=True)
            ready = torch.cuda.Event()
            ready.record(self.side)
        return ready

    def _take(self, ready):
        """Wait (on the device) for the staged batch and copy it into the step's static inputs."""
        cur = torch.cuda.current_stream(self.device)
        cur.wait_event(ready)
        if self.inputs is None:
            self.inputs = {k: torch.empty_like(v) for k, v in self.staging.items()}
        for k, v in self.staging.items():
            self.inputs[k].copy_(v)
        self._consumed.record(cur)

    # -- the step ------------------------------------------------------------------------------------------------------
    def _body(self):
        self.sums += _stats(train_step(self.model, self.optimizer, self.inputs, self.precision)).double()

    def _step(self):
        if self.graph is not None:
            self.graph.replay()
        elif self._eager_steps < WARMUP_STEPS:
            self._body()
            self._eager_steps += 1
        else:
            self.optimizer.zero_grad(set_to_none=True)
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph):
                self._body()
            self.graph.replay()                            # capturing records the step; replaying runs it
        self.step_count += 1

    # -- epochs --------------------------------------------------------------------------------------------------------
    def _read_sums(self, n):
        v = (self.sums / max(n, 1)).tolist()
        self.sums.zero_()
        losses = dict(zip(LOSS_KEYS, v[:3]))
        acc = dict(zip(ACCURACY_KEYS, v[3:]))
        if not self.model.fine:
            del losses["fine"], acc["fine_accuracy"]
        return losses, acc

    def train_epoch(self, epoch):
        """One epoch of steps, batch k + 1 assembled on the side stream while step k runs.  Returns the mean train
        losses and accuracies since the last print."""
        order = epoch_order(self.n_train, self.batch_size, self.seed, epoch)
        seed, rng = batch_draws(self.seed, epoch, 0)
        ready = self._load(order[0], seed, rng, self.make_train)
        since, t0 = 0, time.perf_counter()
        for b in range(len(order)):
            self._take(ready)
            self._step()
            since += 1
            if b + 1 < len(order):
                seed, rng = batch_draws(self.seed, epoch, b + 1)
                ready = self._load(order[b + 1], seed, rng, self.make_train)
            if b % self.print_interval == 0 and b > 0:
                losses, acc = self._read_sums(since)
                t1 = time.perf_counter()
                self.log(format_losses(losses, acc, (t1 - t0) / (since * self.batch_size), self.model.fine))
                since, t0 = 0, t1
        return self._read_sums(since)

    def test(self, epoch):
        """test_model over the whole val list in order, the last partial batch kept; returns (losses, accuracies)
        as means weighted by the batch size."""
        model = self.model
        sums = torch.zeros(5, dtype=torch.float64, device=self.device)
        n, t0 = 0, time.perf_counter()
        model.eval()
        try:
            with torch.no_grad():
                for b, items in enumerate(test_batches(self.n_test, self.batch_size)):
                    seed, rng = batch_draws(self.seed, epoch, b, test=True)
                    t = self.make_test(items, seed, rng, None)
                    inp = dict(zip(INPUT_FIELDS, (v.to(self.device, torch.float32) for v in t[:8])))
                    out = _forward_loss(model, inp, self.precision)
                    sums += len(items) * _stats(out).double()
                    n += len(items)
        finally:
            model.train()
        v = weighted_means(dict(enumerate(sums.tolist())), n)
        self.test_time = (time.perf_counter() - t0) / max(n, 1)
        losses, acc = dict(zip(LOSS_KEYS, (v[0], v[1], v[2]))), dict(zip(ACCURACY_KEYS, (v[3], v[4])))
        if not model.fine:
            del losses["fine"], acc["fine_accuracy"]
        return losses, acc

    def run(self, epochs=None):
        """Train from self.epoch up to `epochs` (the trainer's by default); returns the last checkpoint's path."""
        epochs = self.epochs if epochs is None else int(epochs)
        os.makedirs(self.out_dir, exist_ok=True)
        path = None
        for epoch in range(self.epoch, epochs):
            self.train_epoch(epoch)
            losses, acc = self.test(epoch)
            self.log("Test loss and accuracy:")
            self.log(format_losses(losses, acc, self.test_time, self.model.fine))
            if acc["coarse_accuracy"] > self.best:
                self.best = acc["coarse_accuracy"]
                self.log("--- best test coarse accuracy %f" % self.best)
            self.log("Epoch %d done." % epoch)
            new_lr = decayed_lr(self.lr, epoch, self.lr_decay_step)
            if new_lr != self.lr:
                self.log("update detector learning rate: %f -> %f" % (self.lr, new_lr))
                self._set_lr(new_lr)
            self.log("Saving network...")
            path = os.path.join(self.out_dir, checkpoint_name(self.version, self.gpu, epoch, acc["coarse_accuracy"]))
            torch.save(self.model.state_dict(), path)
            save_resume(os.path.join(self.out_dir, "resume.pth"), self.model, self.optimizer, epoch, self.step_count,
                        self.lr, self.seed, dict(best=self.best, dataset=self.dataset, version=self.version,
                                                 batch_size=self.batch_size,
                                                 point_chain_state=self.model.point_chain_state.cpu()))
            self.epoch = epoch + 1
        return path
