"""KITTI odometry classifier batches from a dataset root: the host code of data/kitti_pc_img_pose_loader.py (the
calibration parse of data/kitti_helper.py KittiCalibHelper, make_kitti_dataset, get_sequence_j,
search_for_accumulation's Pc^-1 P_ij Pc chain) restated, with the points assembled on the device by
assemble.assemble_batch(**kitti_args) from a ScanStore and the images by imageprep.assemble_images.

The float32 roundings and the np.dot / np.linalg.inv calls are the loader's, in its order, so every matrix is the
loader's bit for bit on the same numpy.  Draws (the image pairing j, Pr, the image crop and jitter) come from a numpy
Generator and match the loader in distribution (DESIGN.md 4.11, 4.22).
"""
import os

import numpy as np
import torch

from . import assemble, imageprep

SKIP_START_END = 40                 # make_kitti_dataset
TRAIN_SEQS = tuple(range(9))
VAL_SEQS = (9, 10)
ACCUMULATION_FRAME_NUM = 3          # kitti/options.py
ACCUMULATION_FRAME_SKIP = 6
DELTA_IJ_MAX = 40
TRANSLATION_MAX = 10.0
RECORD_DIR = "voxel0.1-SNr0.6"


def _require(path, what):
    if not os.path.exists(path):
        raise FileNotFoundError(f"KITTI {what} not found: {path}")
    return path


def calib_path(root, seq):
    return os.path.join(root, "calib", "%02d" % seq, "calib.txt")


def pose_path(root, seq, i):
    return os.path.join(root, "poses", "%02d" % seq, "%06d.npz" % i)


def _record_folder(root, seq, name):
    return os.path.join(root, "data_odometry_velodyne_NWU", "sequences", "%02d" % seq, name)


def record_dir(root, seq, record_dir=RECORD_DIR):
    """The sequence's folder of scan records named `record_dir`: the prepared scans (voxel0.1-SNr0.6) by default, or
    e.g. the accumulated frames kitti_build writes (stride4-acc50-voxel0.4)."""
    return _record_folder(root, seq, record_dir)


def record_path(root, seq, i, record_dir=RECORD_DIR):
    return os.path.join(_record_folder(root, seq, record_dir), "%06d.npy" % i)


def image_dirs(root, seq, key):
    """The two folders a sequence's camera frames may be in: the .npy conversion (kitti_png_to_npy.py's output, the
    loader's layout) and KITTI's official .png layout."""
    cam = "image_" + key[1]
    return (os.path.join(root, "data_odometry_color_npy", "sequences", "%02d" % seq, cam),
            os.path.join(root, "data_odometry_color", "sequences", "%02d" % seq, cam))


def image_dir(root, seq, key):
    """The sequence's frame folder: the .npy folder when it exists, otherwise the official PNG folder; raises
    FileNotFoundError naming both when neither exists."""
    npy, png = image_dirs(root, seq, key)
    if os.path.isdir(npy):
        return npy
    if os.path.isdir(png):
        return png
    raise FileNotFoundError(f"KITTI image folder not found: neither {npy} nor {png}")


def image_path(root, seq, key, i):
    """Frame i of the camera: <frame>.npy in the .npy folder when it exists, otherwise <frame>.png."""
    d = image_dir(root, seq, key)
    return os.path.join(d, "%06d.%s" % (i, "npy" if d == image_dirs(root, seq, key)[0] else "png"))


def parse_calib(text, path="calib.txt"):
    """KittiCalibHelper.read_calib_files for one calib.txt: each line 'K: 12 numbers' goes through float32.  Tr becomes
    a float64 4 x 4 [mat; 0 0 0 1]; every other key P gives P_K (the float32 3 x 3) and P, a float64 identity whose
    translation is (tx, ty, tz) recovered in float32 from the 3 x 4 (tz = m23, tx = (m03 - cx tz) / fx, ty = (m13 -
    cy tz) / fy)."""
    out = {}
    for n, line in enumerate(text.splitlines()):
        if not line.strip():
            continue
        key = line[0:2]
        vals = line[4:].split()
        if len(vals) != 12:
            raise ValueError(f"{path}:{n + 1}: expected 'KEY: 12 numbers' (got {line!r})")
        mat = np.array([float(v) for v in vals]).reshape((3, 4)).astype(np.float32)
        if key == "Tr":
            P = np.identity(4)
            P[0:3, :] = mat
            out[key] = P
        else:
            K = mat[0:3, 0:3]
            out[key + "_K"] = K
            fx, fy, cx, cy = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
            tz = mat[2, 3]
            tx = (mat[0, 3] - cx * tz) / fx
            ty = (mat[1, 3] - cy * tz) / fy
            P = np.identity(4)
            P[0:3, 3] = np.asarray([tx, ty, tz])
            out[key] = P
    return out


def read_calib(root, seq):
    path = _require(calib_path(root, seq), "calibration")
    with open(path) as f:
        return parse_calib(f.read(), path)


def camera_Pc(calib, key):
    """The loader's Pc = np.dot(P_key, Tr) (camera key <- velodyne)."""
    for k in (key, "Tr"):
        if k not in calib:
            raise KeyError(f"calibration has no {k!r} entry")
    return np.dot(calib[key], calib["Tr"])


def mode_seqs(mode):
    if mode == "train":
        return TRAIN_SEQS
    if "val" in mode:
        return VAL_SEQS
    raise ValueError(f"KITTI has train and val* modes (got {mode!r})")


def sequence_length(root, seq):
    """The loader's sample count: the number of entries of the sequence's image_2 folder (the one image_dir picks)."""
    d = _require(image_dir(root, seq, "P2"), "image folder")
    n = len(os.listdir(d))
    if n == 0:
        raise ValueError(f"KITTI sequence {seq:02d} is empty: no frame in {d}")
    return n


def make_dataset(root, mode, seqs=None):
    """make_kitti_dataset: for each sequence (0-8 in train, 9 and 10 in any val mode, or `seqs`) and each frame i in
    [40, n - 40), the entries (seq, i, n, 'P2') and (seq, i, n, 'P3'), interleaved."""
    seqs = mode_seqs(mode) if seqs is None else tuple(int(s) for s in seqs)
    out = []
    for seq in seqs:
        n = sequence_length(root, seq)
        for i in range(SKIP_START_END, n - SKIP_START_END):
            out.append((seq, i, n, "P2"))
            out.append((seq, i, n, "P3"))
    if not out:
        raise ValueError(f"the KITTI {mode} list of {root} is empty "
                         f"(every sequence has <= {2 * SKIP_START_END} frames)")
    return out


def accumulation_walk(i, n, frame_num=ACCUMULATION_FRAME_NUM, skip=ACCUMULATION_FRAME_SKIP):
    """get_accumulated_pc's frame order: the anchor i, then i - skip, i - 2 skip, ... and i + skip, i + 2 skip, ...,
    frame_num of each unless the sequence [0, n) ends first."""
    out = [i]
    for stride in (-skip, skip):
        for c in range(1, frame_num + 1):
            j = i + stride * c
            if j < 0 or j >= n:
                break
            out.append(j)
    return out


class KittiDataset:
    """A KITTI root in the loader's layout: the entry list of `mode` (make_dataset), and the calibration and poses
    (float32, as the loader reads them), read once and kept.  record_dir names the folder of scan records the batches
    read (the loader's np_folder)."""

    def __init__(self, root, mode, seqs=None, record_dir=RECORD_DIR):
        self.root = root
        self.mode = mode
        self.record_dir = record_dir
        self.entries = make_dataset(root, mode, seqs)
        self._calib, self._poses, self._inverses = {}, {}, {}

    def __len__(self):
        return len(self.entries)

    def calib(self, seq):
        if seq not in self._calib:
            self._calib[seq] = read_calib(self.root, seq)
        return self._calib[seq]

    def pose(self, seq, i):
        """np.load(poses/%02d/%06d.npz)['pose'].astype(np.float32)."""
        k = (seq, i)
        if k not in self._poses:
            with np.load(_require(pose_path(self.root, seq, i), "pose")) as z:
                self._poses[k] = z["pose"].astype(np.float32)
        return self._poses[k]

    def frame_transforms(self, seq, walk, Pc):
        """frame_T of the walk: the identity for the anchor, then search_for_accumulation's Pc^-1 (P_io P_oj) Pc with
        P_io = inv(P_oi) in float32 and Pc_inv = inv(Pc) in float64."""
        Pc_inv = np.linalg.inv(Pc)
        P_io = np.linalg.inv(self.pose(seq, walk[0]))
        Ts = [np.identity(4)]
        for j in walk[1:]:
            P_ij = np.dot(P_io, self.pose(seq, j))
            Ts.append(np.dot(Pc_inv, np.dot(P_ij, Pc)))
        return np.stack(Ts)

    def pose_inverse(self, seq, i):
        """np.linalg.inv of the float32 pose, computed once per frame."""
        k = (seq, i)
        if k not in self._inverses:
            self._inverses[k] = np.linalg.inv(self.pose(seq, i))
        return self._inverses[k]

    def sequence_j(self, rng, seq, i, n, delta_ij_max=DELTA_IJ_MAX, translation_max=TRANSLATION_MAX):
        """get_sequence_j: j ~ U{max(i - d, 0) .. min(i + d, n - 1)} from rng, redrawn until ||t_ji|| < translation_max,
        with Pji = inv(P_j) P_i in float32.  Only drawn frames are evaluated (their inverses are kept).  A negative
        translation_max gives (i, the float64 identity, 0).  Raises once every frame of the window has been drawn and
        rejected (the loader would draw for ever).  Returns (j, Pji, t_ji)."""
        if translation_max < 0:
            P = np.identity(4)
            return i, P, P[0:3, 3]
        lo, hi = max(i - delta_ij_max, 0), min(i + delta_ij_max, n - 1)
        Pi = self.pose(seq, i)
        rejected = set()
        while len(rejected) < hi - lo + 1:
            j = int(rng.integers(lo, hi + 1))
            if j in rejected:
                continue
            Pji = np.dot(self.pose_inverse(seq, j), Pi)
            if np.linalg.norm(Pji[0:3, 3]) < translation_max:
                return j, Pji, Pji[0:3, 3]
            rejected.add(j)
        raise ValueError(f"KITTI sequence {seq:02d} frame {i}: no frame j in [{lo}, {hi}] lies within "
                         f"translation_max={translation_max} of it")


def read_record(path):
    """A scan record as the loader reads it: np.load(path).astype(np.float32), [7, n] (xyz, intensity, sn)."""
    r = np.load(_require(path, "scan record")).astype(np.float32)
    if r.ndim != 2 or r.shape[0] != 7:
        raise ValueError(f"{path}: a KITTI scan record is [7, n] (got {r.shape})")
    return r


def plan_batch(dataset, items, mode, rng, translation_max=TRANSLATION_MAX, delta_ij_max=DELTA_IJ_MAX):
    """The host half of kitti_batch: per item (an index into dataset.entries) the walk, frame_T, Pc, the drawn j with
    Pji and t_ji, and the raw K, drawing j from rng item by item.  Returns a list of dicts."""
    if mode not in assemble.MODES:
        raise ValueError(f"mode must be one of {assemble.MODES} (got {mode!r})")
    out = []
    for it in items:
        it = int(it)
        if not 0 <= it < len(dataset):
            raise IndexError(f"item {it} is outside the KITTI {dataset.mode} list of {len(dataset)} entries")
        seq, i, n, key = dataset.entries[it]
        cal = dataset.calib(seq)
        Pc = camera_Pc(cal, key)
        walk = accumulation_walk(i, n)
        FT = dataset.frame_transforms(seq, walk, Pc)
        j, Pji, t_ji = dataset.sequence_j(rng, seq, i, n, delta_ij_max, translation_max)
        out.append(dict(seq=seq, i=i, n=n, key=key, walk=walk, frame_T=FT, Pc=Pc, j=j, Pji=Pji, t_ji=t_ji,
                        K=cal[key + "_K"]))
    return out


def scan_store(root, seqs, location="cuda", device=None, record_dir=RECORD_DIR):
    """A long-lived ScanStore of whole sequences (every record of each sequence's record folder, keyed (seq, frame)).
    Opt-in: KITTI sequences 0-8 take tens of GB (DESIGN.md 4.22); store_nbytes gives the size without loading."""
    recs, keys = [], []
    for seq in seqs:
        for name, path in _record_files(root, seq, record_dir):
            recs.append(np.load(path, mmap_mode="r"))
            keys.append((int(seq), int(name[:6])))
    for (seq, i), r in zip(keys, recs):
        if r.ndim != 2 or r.shape[0] != 7:
            raise ValueError(f"{record_path(root, seq, i, record_dir)}: a KITTI scan record is [7, n] (got {r.shape})")
    return assemble.ScanStore(recs, location, keys=keys, device=device)


def _record_files(root, seq, record_dir=RECORD_DIR):
    d = _require(_record_folder(root, seq, record_dir), "scan record folder")
    names = sorted(f for f in os.listdir(d) if f.endswith(".npy"))
    if not names:
        raise ValueError(f"KITTI sequence {seq:02d} is empty: no scan record in {d}")
    return [(f, os.path.join(d, f)) for f in names]


def store_nbytes(root, seqs, record_dir=RECORD_DIR):
    """The bytes a scan_store of `seqs` would take (28 per point: 7 float32 planes), from the .npy headers only."""
    return sum(28 * int(np.load(p, mmap_mode="r").shape[1]) for seq in seqs
               for _, p in _record_files(root, seq, record_dir))


def kitti_batch(root, items, mode, seed, rng=None, store=None, input_pt_num=assemble.INPUT_PT_NUM,
                node_a_num=assemble.NODE_NUM, node_b_num=assemble.NODE_NUM, translation_max=TRANSLATION_MAX,
                delta_ij_max=DELTA_IJ_MAX, device="cuda", stream=None, record_dir=None):
    """KittiLoader.__getitem__ for S = len(items) entries of a KittiDataset (or of KittiDataset(root, mode) when root
    is a path).  j is drawn per item from rng (a numpy Generator or a seed), which then draws Pr and the image crop and
    jitter; seed keys the device's Philox draws.  The scan records come from `store` (a ScanStore keyed (seq, frame),
    e.g. scan_store) or, without one, from a per-batch store of the batch's distinct records, read from the folder
    `record_dir` (None: the dataset's, by default voxel0.1-SNr0.6).  The image is frame j's.
    Returns (pc [S,3,N], intensity [S,1,N], sn [S,3,N], node_a [S,3,Ma], node_b [S,3,Mb], P [S,3,4],
    img [S,3,160,512] float32 on the device; K [S,3,3], t_ji [S,3] float32 on the host)."""
    ds = root if isinstance(root, KittiDataset) else KittiDataset(root, mode)
    items = list(items)
    if not items:
        raise ValueError("items is empty")
    rng = rng if isinstance(rng, np.random.Generator) else np.random.default_rng(rng)
    plan = plan_batch(ds, items, mode, rng, translation_max, delta_ij_max)
    keys = [(p["seq"], j) for p in plan for j in p["walk"]]
    fs = np.concatenate([[s] * len(p["walk"]) for s, p in enumerate(plan)])
    FT = np.concatenate([p["frame_T"] for p in plan])
    if store is not None:
        frames = assemble.store_frames(store, [store.index(k) for k in keys], fs, FT)
    else:
        uniq, ids = assemble.unique_records(keys)
        folder = ds.record_dir if record_dir is None else record_dir
        recs = [read_record(record_path(ds.root, seq, i, folder)) for seq, i in uniq]
        frames = assemble.batch_frames(recs, ids, fs, FT, device, stream)
    Pc = np.stack([p["Pc"] for p in plan])
    Pji = np.stack([p["Pji"] for p in plan])
    out = assemble.assemble_batch(frames, mode, seed, input_pt_num=input_pt_num, node_a_num=node_a_num,
                                  node_b_num=node_b_num, rng=rng, stream=stream, **assemble.kitti_args(Pc, Pji))
    paths = [_require(image_path(ds.root, p["seq"], p["key"], p["j"]), "image") for p in plan]
    png = [k for k, q in enumerate(paths) if q.endswith(".png")]
    if len(png) == len(paths):
        images = imageprep.read_png_batch(paths, device, stream)
    else:                                   # .npy frames, or sequences of both kinds in one batch
        imgs = [None if k in png else np.load(q) for k, q in enumerate(paths)]
        if png:
            dec = imageprep.read_png_batch([paths[k] for k in png], device, stream)
            data = dec["data"].cpu().numpy()
            for k, o, (h, w) in zip(png, dec["offsets"], dec["shapes"]):
                imgs[k] = data[o:o + 3 * h * w].reshape(h, w, 3)
        images = imageprep.pack_images(imgs, device)
    K = np.stack([p["K"] for p in plan])
    im = imageprep.assemble_images(images, K, mode, rng=rng, flip=out["flip"], stream=stream,
                                   **imageprep.kitti_image_args())
    t_ji = np.stack([np.asarray(p["t_ji"]) for p in plan]).astype(np.float32)
    return (out["pc"], out["intensity"], out["sn"], out["node_a"], out["node_b"], out["P"], im["img"], im["K"],
            torch.from_numpy(t_ji))
