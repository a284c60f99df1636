"""Oxford RobotCar classifier batches from a dataset root: the host code of data/oxford_pc_img_pose_loader.py
(read_train_val_split, make_oxford_dataset with its float32 P_convert conjugation, get_camera_timestamp) restated,
with the points assembled on the device by assemble.assemble_batch(**oxford_args) from a ScanStore and the JPEG
frames decoded and assembled by imageprep.read_jpeg_batch / assemble_images.

Poses and P_cam_pc are the loader's bit for bit on the same numpy; the camera draw, Pr and the image crop and jitter
come from a numpy Generator and match the loader in distribution (DESIGN.md 4.11, 4.22).
"""
import bisect
import math
import os

import numpy as np
import torch

from . import assemble, imageprep

PC_BUILD_INTERVAL = 2               # oxford/options.py
TRANSLATION_MAX = 10.0
TEST_TRANSLATION_MAX = 10.0
PC_MAX_RANGE = 50.0
# data/oxford_pc_img_pose_loader.py:221
K_CENTRE = np.asarray([[964.828979, 0, 643.788025], [0, 964.828979, 484.407990], [0, 0, 1]], dtype=np.float32)
P_CONVERT = np.asarray([[0, 1, 0, 0], [0, 0, 1, 0], [1, 0, 0, 0], [0, 0, 0, 1]], dtype=np.float32)


def _require(path, what):
    if not os.path.exists(path):
        raise FileNotFoundError(f"Oxford {what} not found: {path}")
    return path


def record_path(root, traversal, ts, remove_ground=False):
    return os.path.join(root, traversal, "lms_front_foreground" if remove_ground else "lms_front", "%d.npy" % ts)


def image_path(root, traversal, ts):
    return os.path.join(root, traversal, "stereo", "centre", "%d.jpg" % ts)


def read_split(root, mode):
    """read_train_val_split of train.txt (train) or val.txt (any val mode): one traversal per line."""
    if mode == "train":
        name = "train.txt"
    elif "val" in mode:
        name = "val.txt"
    else:
        raise ValueError(f"Oxford has train and val* modes (got {mode!r})")
    with open(_require(os.path.join(root, name), "split file")) as f:
        out = [x.rstrip() for x in f.readlines()]
    return [t for t in out if t]


def convert_poses(poses):
    """make_oxford_dataset's conjugation: each pose (as float32) -> P_convert (P inv(P_convert)), float32."""
    P = np.array(poses).astype(np.float32)
    P_convert_inv = np.linalg.inv(P_CONVERT)
    for b in range(P.shape[0]):
        P[b] = np.dot(P_CONVERT, np.dot(P[b], P_convert_inv))
    return P


class Traversal:
    """One traversal's pc / camera timestamps (Python lists of ints) and converted float32 poses."""

    def __init__(self, root, name):
        d = os.path.join(root, name)
        self.name = name
        self.pc_timestamps = np.load(_require(os.path.join(d, "pc_timestamps.npy"), "timestamps")).tolist()
        self.pc_poses = convert_poses(np.load(_require(os.path.join(d, "pc_poses.npy"), "poses")))
        self.camera_timestamps = np.load(_require(os.path.join(d, "camera_timestamps.npy"), "timestamps")).tolist()
        self.camera_poses = convert_poses(np.load(_require(os.path.join(d, "camera_poses.npy"), "poses")))
        if len(self.pc_timestamps) == 0:
            raise ValueError(f"Oxford traversal {name} is empty: no point cloud in {d}")
        if len(self.pc_poses) != len(self.pc_timestamps) or len(self.camera_poses) != len(self.camera_timestamps):
            raise ValueError(f"Oxford traversal {name}: one pose per timestamp")
        if len(self.camera_timestamps) == 0:
            raise ValueError(f"Oxford traversal {name} has no camera frame")
        self.camera_inverses = {}          # camera index -> np.linalg.inv of its pose


class OxfordDataset:
    """make_oxford_dataset: the split's traversals and the entries (traversal, pc timestamp, index, pc count)."""

    def __init__(self, root, mode, traversals=None):
        self.root = root
        self.mode = mode
        names = read_split(root, mode) if traversals is None else list(traversals)
        if not names:
            raise ValueError(f"the Oxford {mode} split of {root} lists no traversal")
        self.traversals = {t: Traversal(root, t) for t in names}
        self.entries = []
        for t in names:
            tr = self.traversals[t]
            for i, ts in enumerate(tr.pc_timestamps):
                self.entries.append((t, ts, i, len(tr.pc_timestamps)))

    def __len__(self):
        return len(self.entries)


def camera_index(rng, tr, i, translation_max, pc_build_interval=PC_BUILD_INTERVAL):
    """get_camera_timestamp: the camera window is bisect_left of the pc timestamps ceil(translation_max / interval)
    indices either side of i; cam ~ U{window} from rng, redrawn until ||t|| < translation_max with P_cam_pc =
    inv(P_o_cam) P_o_pc in float32; only drawn frames are evaluated (their inverses are kept).  A draw past the last
    camera frame is redrawn (the loader would index past its list).  Raises once every index of the window has been
    drawn and rejected.  Returns (cam index, P_cam_pc)."""
    n = len(tr.pc_timestamps)
    step = math.ceil(translation_max / pc_build_interval)
    prev_t = tr.pc_timestamps[max(0, i - step)]
    next_t = tr.pc_timestamps[min(n - 1, i + step)]
    lo = bisect.bisect_left(tr.camera_timestamps, prev_t)
    hi = bisect.bisect_left(tr.camera_timestamps, next_t)
    P_o_pc = tr.pc_poses[i]
    rejected = set()
    while len(rejected) < hi - lo + 1:
        c = int(rng.integers(lo, hi + 1))
        if c in rejected:
            continue
        if c < len(tr.camera_timestamps):
            if c not in tr.camera_inverses:
                tr.camera_inverses[c] = np.linalg.inv(tr.camera_poses[c])
            P = np.dot(tr.camera_inverses[c], P_o_pc)
            if np.linalg.norm(P[0:3, 3]) < translation_max:
                return c, P
        rejected.add(c)
    raise ValueError(f"Oxford traversal {tr.name} cloud {i}: no camera frame in [{lo}, {hi}] lies within "
                     f"translation_max={translation_max} of it")


def read_record(path):
    """np.load(path).astype(np.float32), [4, n] (xyz in camera axes, intensity)."""
    r = np.load(_require(path, "scan record")).astype(np.float32)
    if r.ndim != 2 or r.shape[0] != 4:
        raise ValueError(f"{path}: an Oxford scan record is [4, n] (got {r.shape})")
    return r


def plan_batch(dataset, items, mode, rng, translation_max=None):
    """The host half of oxford_batch: per item the traversal, pc timestamp, drawn camera index and P_cam_pc (float32),
    drawing from rng item by item; translation_max defaults to the loader's (train) / test value."""
    if mode not in assemble.MODES:
        raise ValueError(f"mode must be one of {assemble.MODES} (got {mode!r})")
    if translation_max is None:
        translation_max = TRANSLATION_MAX if mode == "train" else TEST_TRANSLATION_MAX
    out = []
    for it in items:
        it = int(it)
        if not 0 <= it < len(dataset):
            raise IndexError(f"item {it} is outside the Oxford {dataset.mode} list of {len(dataset)} entries")
        t, ts, i, _ = dataset.entries[it]
        tr = dataset.traversals[t]
        c, P = camera_index(rng, tr, i, translation_max)
        out.append(dict(traversal=t, pc_timestamp=ts, i=i, cam=c, camera_timestamp=tr.camera_timestamps[c],
                        P_cam_pc=P))
    return out


def scan_store(root, traversals, location="cuda", device=None, remove_ground=False):
    """A long-lived ScanStore of whole traversals (every pc timestamp's record, keyed (traversal, timestamp))."""
    recs, keys = [], []
    for t in traversals:
        ts_path = _require(os.path.join(root, t, "pc_timestamps.npy"), "timestamps")
        for ts in np.load(ts_path).tolist():
            p = _require(record_path(root, t, ts, remove_ground), "scan record")
            r = np.load(p, mmap_mode="r")
            if r.ndim != 2 or r.shape[0] != 4:
                raise ValueError(f"{p}: an Oxford scan record is [4, n] (got {r.shape})")
            recs.append(r)
            keys.append((t, ts))
    return assemble.ScanStore(recs, location, keys=keys, device=device)


def oxford_batch(root, items, mode, seed, rng=None, store=None, input_pt_num=assemble.INPUT_PT_NUM,
                 node_a_num=assemble.NODE_NUM, node_b_num=assemble.NODE_NUM, remove_ground=False, device="cuda",
                 stream=None):
    """OxfordLoader.__getitem__ for S = len(items) entries of an OxfordDataset (or of OxfordDataset(root, mode) when
    root is a path).  The camera frame is drawn per item from rng (a numpy Generator or a seed), which then draws Pr
    and the image crop and jitter; seed keys the device's Philox draws.  Records come from `store` (keyed (traversal,
    timestamp), e.g. scan_store) or from a per-batch store of the batch's distinct records.  Returns (pc [S,3,N],
    intensity [S,1,N], sn [S,3,N] (zeros), node_a, node_b, P [S,3,4], img [S,3,384,640] float32 on the device; K
    [S,3,3], t_ij [S,3] float32 on the host)."""
    ds = root if isinstance(root, OxfordDataset) else OxfordDataset(root, mode)
    items = list(items)
    if not items:
        raise ValueError("items is empty")
    rng = rng if isinstance(rng, np.random.Generator) else np.random.default_rng(rng)
    plan = plan_batch(ds, items, mode, rng)
    keys = [(p["traversal"], p["pc_timestamp"]) for p in plan]
    S = len(plan)
    FT = np.tile(np.identity(4), (S, 1, 1))
    if store is not None:
        frames = assemble.store_frames(store, [store.index(k) for k in keys], np.arange(S), FT)
    else:
        uniq, ids = assemble.unique_records(keys)
        recs = [read_record(record_path(ds.root, t, ts, remove_ground)) for t, ts in uniq]
        frames = assemble.batch_frames(recs, ids, np.arange(S), FT, device, stream)
    P_cam_pc = np.stack([p["P_cam_pc"] for p in plan])
    out = assemble.assemble_batch(frames, mode, seed, input_pt_num=input_pt_num, node_a_num=node_a_num,
                                  node_b_num=node_b_num, rng=rng, stream=stream,
                                  **assemble.oxford_args(P_cam_pc, pc_max_range=PC_MAX_RANGE))
    images = imageprep.read_jpeg_batch([_require(image_path(ds.root, p["traversal"], p["camera_timestamp"]), "image")
                                        for p in plan], device, stream)
    im = imageprep.assemble_images(images, K_CENTRE, mode, rng=rng, stream=stream, **imageprep.oxford_image_args())
    t_ij = P_cam_pc[:, 0:3, 3].astype(np.float32)
    return (out["pc"], out["intensity"], out["sn"], out["node_a"], out["node_b"], out["P"], im["img"], im["K"],
            torch.from_numpy(t_ij))
