"""Build a nuScenes dataroot's dataset_info.list (data/nuscenes/make_datasets.py) from the raw tables, with the camera
walks on the device and without nuscenes-devkit or pyquaternion.

The host reads <dataroot>/<version>/{scene, sample, sample_data, sensor, calibrated_sensor, ego_pose}.json once into
columnar arrays (RawTables), rebuilds the two parts of the devkit's reverse index the script reads (each record's
channel, each sample's key-frame record per channel), filters the scenes, walks the LIDAR_TOP chains with the script's
counter and inverts the kept sweeps' poses with np.linalg.inv.  csrc/nuscenes_build.cu then runs every (entry, camera,
direction) walk; a step it cannot decide exactly is handed back and resumed here with the script's own numpy calls,
so the list equals the script's on the same numpy.  DESIGN.md 4.28 states the contract and marks the devkit
behaviours restated from its documentation and source.
"""
import json
import os
import pickle
import time

import numpy as np
import torch

from . import _native
from ._native import _ptr, _require_cuda
from .nuscenes import CAMERAS, P_from_record

LIDAR = "LIDAR_TOP"
TABLES = ("scene", "sample", "sample_data", "sensor", "calibrated_sensor", "ego_pose")
# make_datasets.py's test_night_scene_tokens: scenes kept out of the list whatever their description says
TEST_NIGHT_SCENE_TOKENS = (
    "e59a4d0cc6a84ed59f78fb21a45cdcb4", "7209495d06f24712a063ac6c4a9b403b", "3d776ea805f240bb925bd9b50b258416",
    "48f81c548d0148fc8010a73d70b2ef9c", "2ab683f384234dce89800049dec19a30", "7edca4c44eac4f52a3105e1794e56b7e",
    "81c939ce8c0d4cc7b159cb5ed4c4e712", "24e6e64ecf794be4a51f7454c8b6d0b2", "828ed34a5e0c456fbf0751cabbab3341",
    "edfd6cfd1805477fbeadbd29f39ed599", "7692a3e112b44b408d191e45954a813c", "58d27a9f83294d99a4ff451dcad5f4d2",
    "a1573aef0bf74324b373dd8a22b4dd68", "ba06095d4e2e425b8e398668abc301d8", "7c315a1db2ac49439d281605f3cca6be",
    "732d7a84353f4ada803a9a115728496c", "1630a1d9cf8a46b3843662a23126e3f6", "f437809584344859882bdff7f8784c43")
NONE, DANGLING = -1, -2             # an empty link, a token that names no record
WALK_DONE, WALK_DEFERRED, WALK_BAD_LINK, WALK_CYCLE = 0, 1, 2, 3      # DIB_NSW_* of include/deepi2p_b200.h
GAMMA4 = 4.440892098500632e-16      # csrc/nuscenes_build.cu's kGamma4: 4u / (1 - 4u), u = 2^-53, rounded up


def deferral_bound(s, n):
    """The device's bound on |N_numpy - N| for a step with sum |inv_ij p_j| = s and norm n (DESIGN.md 4.28)."""
    return 4.0 * GAMMA4 * (s + n)


def _index(tokens):
    """token -> row, the last row winning for a repeated token as in the devkit's _token2ind."""
    return {t: i for i, t in enumerate(tokens)}


def _links(tokens, index):
    return np.array([NONE if t == "" else index.get(t, DANGLING) for t in tokens], dtype=np.int32)


class RawTables:
    """The six tables as columns.  Tokens stay Python lists (the output names records by token); links and indices are
    int32 (NONE for '', DANGLING for a token no record has), translations float32 (the script's cast), rotations
    float64 as read.

    scene_token, scene_description, scene_first (sample row);  sample_token, sample_data [n_sample, n_channel] (the
    key-frame sample_data row per channel, NONE when absent);  channels (the sensor table's channel names);
    sd_token, sd_next, sd_prev, sd_ego, sd_sample, sd_channel, sd_key;  ego_translation [n, 3], ego_rotation [n, 4]."""

    def __init__(self, dataroot, version):
        self.dataroot, self.version = dataroot, version
        t0 = time.perf_counter()
        raw = {}
        for name in TABLES:
            path = os.path.join(dataroot, version, name + ".json")
            if not os.path.isfile(path):
                raise FileNotFoundError(f"no {name} table at {path}")
            with open(path) as f:
                raw[name] = json.load(f)
        self.parse_seconds = time.perf_counter() - t0
        t0 = time.perf_counter()
        sensor, calib, ego = raw["sensor"], raw["calibrated_sensor"], raw["ego_pose"]
        sample, sd, scene = raw["sample"], raw["sample_data"], raw["scene"]
        self.channels = list(dict.fromkeys(r["channel"] for r in sensor))
        ch_of = {c: k for k, c in enumerate(self.channels)}
        sensor_ch = {r["token"]: ch_of[r["channel"]] for r in sensor}
        calib_ch = {}
        for r in calib:
            if r["sensor_token"] not in sensor_ch:
                raise ValueError(f"calibrated_sensor {r['token']}: no sensor {r['sensor_token']!r}")
            calib_ch[r["token"]] = sensor_ch[r["sensor_token"]]
        self.ego_token = [r["token"] for r in ego]
        ego_index = _index(self.ego_token)
        self.ego_translation = np.array([r["translation"] for r in ego], dtype=np.float64).reshape(-1, 3).astype(
            np.float32)
        self.ego_rotation = np.array([r["rotation"] for r in ego], dtype=np.float64).reshape(-1, 4)
        self.sample_token = [r["token"] for r in sample]
        sample_index = _index(self.sample_token)
        self.sd_token = [r["token"] for r in sd]
        self.sd_index = _index(self.sd_token)
        self.sd_next = _links([r["next"] for r in sd], self.sd_index)
        self.sd_prev = _links([r["prev"] for r in sd], self.sd_index)
        self.sd_ego = _links([r["ego_pose_token"] for r in sd], ego_index)
        self.sd_sample = _links([r["sample_token"] for r in sd], sample_index)
        self.sd_key = np.array([bool(r["is_key_frame"]) for r in sd], dtype=bool)
        try:
            self.sd_channel = np.array([calib_ch[r["calibrated_sensor_token"]] for r in sd], dtype=np.int32)
        except KeyError as e:
            raise ValueError(f"a sample_data record names no calibrated_sensor {e.args[0]!r}") from None
        # the devkit's reverse index: sample['data'][channel] = token over the key frames in table order, the last
        # record winning where two compete
        key = np.flatnonzero(self.sd_key)
        bad = key[self.sd_sample[key] < 0]
        if bad.size:
            raise ValueError(f"key-frame sample_data {self.sd_token[bad[0]]} names no sample")
        nc = len(self.channels)
        self.sample_data = np.full((len(sample), nc), NONE, dtype=np.int32)
        slot = self.sd_sample[key].astype(np.int64) * nc + self.sd_channel[key]
        u, first_rev = np.unique(slot[::-1], return_index=True)
        self.sample_data.reshape(-1)[u] = key[::-1][first_rev]
        self.scene_token = [r["token"] for r in scene]
        self.scene_description = [r["description"] for r in scene]
        self.scene_first = _links([r["first_sample_token"] for r in scene], sample_index)
        self.index_seconds = time.perf_counter() - t0

    def channel(self, name):
        return self.channels.index(name) if name in self.channels else None

    def ego_record(self, sd):
        """The ego_pose of sample_data row sd as the dict P_from_record reads."""
        e = int(self.sd_ego[sd])
        if e < 0:
            raise ValueError(f"sample_data {self.sd_token[sd]} names no ego_pose")
        return dict(rotation=self.ego_rotation[e], translation=self.ego_translation[e])


def daytime_scenes(tables):
    """get_lidar_token_list's filter: scene rows in table order, without those whose description contains 'night' or
    'Night' and those in TEST_NIGHT_SCENE_TOKENS."""
    return [i for i, (t, d) in enumerate(zip(tables.scene_token, tables.scene_description))
            if not ("night" in d or "Night" in d or t in TEST_NIGHT_SCENE_TOKENS)]


def scene_lidar_rows(tables, scene, frame_skip):
    """get_scene_lidar_token: the first sample's LIDAR_TOP record, then along next the records where a counter that
    starts at 1 and is incremented before the test is a multiple of frame_skip (chain positions 0, s - 1, 2 s - 1,
    ...)."""
    first = int(tables.scene_first[scene])
    if first < 0:
        raise ValueError(f"scene {tables.scene_token[scene]} names no first sample")
    ch = tables.channel(LIDAR)
    lidar = NONE if ch is None else int(tables.sample_data[first, ch])
    if lidar < 0:
        raise ValueError(f"sample {tables.sample_token[first]} has no {LIDAR} record")
    nxt = tables.sd_next
    out, counter = [lidar], 1
    for _ in range(len(nxt)):
        lidar = int(nxt[lidar])
        if lidar == NONE:
            return out
        if lidar < 0:
            raise ValueError(f"a {LIDAR} record of scene {tables.scene_token[scene]} links to no record")
        counter += 1
        if counter % frame_skip == 0:
            out.append(lidar)
    raise ValueError(f"the {LIDAR} chain of scene {tables.scene_token[scene]} has a cycle")


def plan(tables, frame_skip=2):
    """The entries: kept LIDAR_TOP rows over the daytime scenes, their key-frame record per camera (own [E, 6]) and
    the inverse of each sweep's pose (inv [E, 4, 4], one np.linalg.inv call on the stack)."""
    if int(frame_skip) != frame_skip or frame_skip < 1:
        raise ValueError(f"frame_skip must be a positive integer (got {frame_skip!r})")
    scenes = daytime_scenes(tables)
    rows = [r for s in scenes for r in scene_lidar_rows(tables, s, int(frame_skip))]
    lidar = np.array(rows, dtype=np.int64)
    own = np.empty((len(rows), len(CAMERAS)), dtype=np.int32)
    cams = [tables.channel(c) for c in CAMERAS]
    Ps, cache = [], {}
    for e, r in enumerate(rows):
        s = int(tables.sd_sample[r])
        if s < 0:
            raise ValueError(f"sample_data {tables.sd_token[r]} names no sample")
        for k, ch in enumerate(cams):
            own[e, k] = NONE if ch is None else tables.sample_data[s, ch]
            if own[e, k] < 0:
                raise ValueError(f"sample {tables.sample_token[s]} has no {CAMERAS[k]} record")
        eg = int(tables.sd_ego[r])
        if eg not in cache:
            cache[eg] = P_from_record(tables.ego_record(r))          # get_sample_data_ego_pose_P
        Ps.append(cache[eg])
    inv = np.linalg.inv(np.stack(Ps)) if rows else np.zeros((0, 4, 4))
    return dict(scenes=scenes, lidar=lidar, own=own, inv=inv)


def walk_host(tables, inv, cur, direction, max_translation, out):
    """search_nearby_cameras from the record whose `direction` link gives the next candidate: appends to out while
    norm(dot(inv, P_c)[0:3, 3]) < max_translation, with the script's numpy calls, and stops at the first failure or
    the chain's end."""
    link = tables.sd_next if direction == "next" else tables.sd_prev
    for _ in range(len(link)):
        cand = int(link[cur])
        if cand == NONE:
            return out
        if cand < 0:
            raise ValueError(f"sample_data {tables.sd_token[cur]}: its {direction} names no record")
        camera_P = P_from_record(tables.ego_record(cand))
        t_lc = np.dot(inv, camera_P)[0:3, 3]
        if np.linalg.norm(t_lc) < max_translation:
            out.append(cand)
            cur = cand
        else:
            return out
    raise ValueError(f"the {direction} chain from sample_data {tables.sd_token[cur]} has a cycle")


def walks_host(tables, p, max_translation):
    """Every walk on the host (the rule the device defers to): [E][6] lists of rows, own first, then next, then
    prev."""
    out = []
    for e in range(len(p["lidar"])):
        per = []
        for k in range(len(CAMERAS)):
            own = int(p["own"][e, k])
            rows = [own]
            for d, link in (("next", tables.sd_next), ("prev", tables.sd_prev)):
                first = int(link[own])
                if first >= 0:
                    walk_host(tables, p["inv"][e], first, d, max_translation, rows)
                elif first != NONE:
                    raise ValueError(f"sample_data {tables.sd_token[own]}: its {d} names no record")
            per.append(rows)
        out.append(per)
    return out


def walks_device(tables, p, max_translation, device="cuda", stream=None):
    """The count, scan and fill passes on the device.  Returns dict(counts [W] i32, status [W] i32, offsets [W + 1]
    i64, tokens [total] i32, all host numpy, lane w = 2 (6 e + c) + d, and seconds: CUDA events around the three
    passes and the read of the total between them)."""
    _require_cuda()
    lib = _native.load()
    max_translation = float(max_translation)
    if not np.isfinite(max_translation) or max_translation < 0:
        raise ValueError(f"max_translation must be finite and >= 0 (got {max_translation})")
    dev = torch.device(device)
    st = stream if stream is not None else torch.cuda.current_stream(dev)
    with torch.cuda.stream(st):
        return _walks_on(lib, tables, p, max_translation, dev, st)


def _walks_on(lib, tables, p, max_translation, dev, st):
    E = len(p["lidar"])
    W = 12 * E
    cuda = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    trans = np.full((len(tables.sd_token), 3), np.nan, dtype=np.float32)
    known = tables.sd_ego >= 0                 # an unknown ego pose is deferred, and the host names the record
    trans[known] = tables.ego_translation[tables.sd_ego[known]]
    nxt, prv, tr = cuda(tables.sd_next), cuda(tables.sd_prev), cuda(trans)
    own = cuda(p["own"])
    inv = cuda(np.ascontiguousarray(p["inv"][:, 0:3, :]).reshape(E, 12))
    counts = torch.empty(W, dtype=torch.int32, device=dev)
    status = torch.empty(W, dtype=torch.int32, device=dev)
    offsets = torch.empty(W + 1, dtype=torch.int64, device=dev)
    ws = torch.empty(max(1, lib.nuscenes_walk_scan_workspace_bytes(W) // 8), dtype=torch.int64, device=dev)
    sp = st.cuda_stream
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record(st)
    n_sd = len(tables.sd_token)
    _native.check(lib.nuscenes_walk_count(_ptr(nxt), _ptr(prv), _ptr(tr), n_sd, _ptr(own), _ptr(inv), E,
                                          max_translation, _ptr(counts), _ptr(status), sp), "nuscenes_walk_count")
    _native.check(lib.nuscenes_walk_scan(_ptr(counts), W, _ptr(offsets), _ptr(ws), ws.numel() * 8, sp),
                  "nuscenes_walk_scan")
    total = int(offsets[W].item())
    tokens = torch.empty(max(total, 1), dtype=torch.int32, device=dev)
    if total:
        _native.check(lib.nuscenes_walk_fill(_ptr(nxt), _ptr(prv), _ptr(tr), n_sd, _ptr(own), _ptr(inv), E,
                                             max_translation, _ptr(offsets), _ptr(tokens), sp), "nuscenes_walk_fill")
    ev[1].record(st)
    res = dict(counts=counts.cpu().numpy(), status=status.cpu().numpy(), offsets=offsets.cpu().numpy(),
               tokens=tokens[:total].cpu().numpy())
    ev[1].synchronize()
    res["seconds"] = ev[0].elapsed_time(ev[1]) / 1e3
    return res


def resolve(tables, p, walks, max_translation):
    """The device's walks as [E][6] row lists (own, next, prev), each deferred walk resumed on the host from its
    undecided step.  Returns (lists, number of deferred walks)."""
    status, counts, off, tok = walks["status"], walks["counts"], walks["offsets"], walks["tokens"]
    bad = np.flatnonzero((status == WALK_BAD_LINK) | (status == WALK_CYCLE))
    if bad.size:
        w = int(bad[0])
        e, k, d = w // 12, (w // 2) % 6, ("next", "prev")[w & 1]
        what = "links to no record" if status[w] == WALK_BAD_LINK else "has a cycle"
        raise ValueError(f"the {d} chain of {CAMERAS[k]} from sample_data "
                         f"{tables.sd_token[int(p['own'][e, k])]} {what}")
    own = p["own"]
    tl = tok.tolist()
    out = []
    for e in range(len(p["lidar"])):
        per = []
        for k in range(len(CAMERAS)):
            rows = [int(own[e, k])]
            for d in (0, 1):
                w = 2 * (6 * e + k) + d
                rows += tl[off[w]:off[w + 1]]
                if status[w] == WALK_DEFERRED:
                    link = tables.sd_prev if d else tables.sd_next
                    cur = rows[-1] if counts[w] else int(link[rows[0]])
                    walk_host(tables, p["inv"][e], cur, ("next", "prev")[d], max_translation, rows)
            per.append(rows)
        out.append(per)
    return out, int((status == WALK_DEFERRED).sum())


def to_list(tables, p, rows):
    """[(lidar_token, {camera: [tokens]})] in the script's order."""
    tok = tables.sd_token
    return [(tok[int(r)], {c: [tok[i] for i in cr] for c, cr in zip(CAMERAS, per)})
            for r, per in zip(p["lidar"], rows)]


def make_dataset_info(dataroot, version, frame_skip=2, max_translation=10.0, device="cuda", stream=None,
                      stats=None):
    """make_nuscenes_dataset for <dataroot>/<version>, pickled to <dataroot>/dataset_info.list as the script writes
    it.  Returns the list.  A dict passed as stats receives the counts and each stage's seconds."""
    _require_cuda()
    t0 = time.perf_counter()
    tables = RawTables(dataroot, version)
    t1 = time.perf_counter()
    p = plan(tables, frame_skip)
    t2 = time.perf_counter()
    walks = walks_device(tables, p, max_translation, device, stream)
    t3 = time.perf_counter()
    rows, deferred = resolve(tables, p, walks, max_translation)
    items = to_list(tables, p, rows)
    with open(os.path.join(dataroot, "dataset_info.list"), "wb") as f:
        pickle.dump(items, f)
    t4 = time.perf_counter()
    if stats is not None:
        stats.update(entries=len(items), scenes=len(p["scenes"]), scenes_total=len(tables.scene_token),
                     sample_data=len(tables.sd_token), walks=12 * len(items), deferred=deferred,
                     tokens=int(walks["offsets"][-1]), json_seconds=tables.parse_seconds,
                     index_seconds=tables.index_seconds, plan_seconds=t2 - t1, device_seconds=walks["seconds"],
                     walk_seconds=t3 - t2, assemble_seconds=t4 - t3, total_seconds=t4 - t0)
    return items
