"""Per-entry numpy restatement of data/nuscenes/make_datasets.py's make_nuscenes_dataset, for the tests and the bench
only.  Devkit stands in for nuscenes.nuscenes.NuScenes with a dict per record, as the devkit holds them (DESIGN.md
4.28 marks the rules restated from its documentation and source): .scene, .get(table, token), each sample_data
record's 'channel' through calibrated_sensor -> sensor, and sample['data'][channel] over the key frames in table
order.  make_dataset then runs the script's loop: lidar tokens, per entry one np.linalg.inv, per camera step one
np.dot and one np.linalg.norm.
"""
import json
import os

import numpy as np

from deepi2p_b200.nuscenes import CAMERAS, P_from_record
from deepi2p_b200.nuscenes_build import TABLES, TEST_NIGHT_SCENE_TOKENS


class Devkit:
    def __init__(self, version="v1.0-mini", dataroot=None, verbose=False):
        self.version, self.dataroot = version, dataroot
        self._t, self._ind = {}, {}
        for name in TABLES:
            with open(os.path.join(dataroot, version, name + ".json")) as f:
                self._t[name] = json.load(f)
            self._ind[name] = {r["token"]: i for i, r in enumerate(self._t[name])}
        for r in self._t["sample_data"]:
            cs = self.get("calibrated_sensor", r["calibrated_sensor_token"])
            r["channel"] = self.get("sensor", cs["sensor_token"])["channel"]
        for r in self._t["sample"]:
            r["data"] = {}
        for r in self._t["sample_data"]:
            if r["is_key_frame"]:
                self.get("sample", r["sample_token"])["data"][r["channel"]] = r["token"]

    @property
    def scene(self):
        return self._t["scene"]

    def get(self, table, token):
        return self._t[table][self._ind[table][token]]


def lidar_tokens(nusc, frame_skip):
    out = []
    for scene in nusc.scene:
        d = scene["description"]
        if "night" in d or "Night" in d or scene["token"] in TEST_NIGHT_SCENE_TOKENS:
            continue
        lidar = nusc.get("sample_data", nusc.get("sample", scene["first_sample_token"])["data"]["LIDAR_TOP"])
        out.append(lidar["token"])
        counter = 1
        while lidar["next"] != "":
            lidar = nusc.get("sample_data", lidar["next"])
            counter += 1
            if counter % frame_skip == 0:
                out.append(lidar["token"])
    return out


def ego_P(nusc, sd):
    return P_from_record(nusc.get("ego_pose", sd["ego_pose_token"]))


def entry(nusc, lidar_token, max_translation):
    """(lidar_token, {camera: [tokens]}) for one kept sweep."""
    lidar = nusc.get("sample_data", lidar_token)
    inv = np.linalg.inv(ego_P(nusc, lidar))
    sample = nusc.get("sample", lidar["sample_token"])
    cams = {}
    for name in CAMERAS:
        own = nusc.get("sample_data", sample["data"][name])
        toks = [own["token"]]
        for d in ("next", "prev"):
            if own[d] == "":
                continue
            cam = nusc.get("sample_data", own[d])
            while cam[d] != "":
                tok = cam[d]
                cam = nusc.get("sample_data", tok)
                if np.linalg.norm(np.dot(inv, ego_P(nusc, cam))[0:3, 3]) < max_translation:
                    toks.append(tok)
                else:
                    break
        cams[name] = toks
    return lidar_token, cams


def make_dataset(nusc, frame_skip=2, max_translation=10.0, limit=None):
    toks = lidar_tokens(nusc, frame_skip)
    return [entry(nusc, t, max_translation) for t in (toks if limit is None else toks[:limit])]
