"""Waymo reader with the reference's class and method names (datasets/waymo_data.py:22-208).  Like the reference it starts from
the per-category tracklet index `sot_infos_<category>_<split>.pkl` ({tracklet name: [{"PC": path of the frame's lidar pickle,
"Box": [cx, cy, cz, l, w, h, vx, vy, heading], "Class": name}, ...]}) and the converter's per-frame pickles
(`lidar/...pkl` with `lidars.points_xyz`, `annos/...pkl` with the 4x4 `veh_to_global`); producing those from the raw
tfrecords is the reference's offline conversion script (datasets/generate_waymo_sot.py) and is out of scope here — a missing
index raises FileNotFoundError instead of starting a conversion.

Per frame (waymo_data.py:121-168): points vehicle -> global with `veh_to_global`; the box is built in the vehicle frame with
width / length swapped into the (w, l, h) order and a rotation of -heading about z (Waymo measures heading clockwise from +x in
this convention), then rotated and translated into the global frame."""
import os
import pickle
import re

import numpy as np

from .data_classes import Box, PointCloud
from .kitti import BaseDataset, _rotz


class WaymoDataset(BaseDataset):
    def __init__(self, path, split, category_name="VEHICLE", **kwargs):
        super().__init__(path, split, category_name, **kwargs)
        self.Waymo_Folder = path
        self.split = 'val' if split.lower() == 'test' else split.lower()
        self.category_name = category_name.lower()
        assert self.split in ('train', 'val') and self.category_name in ('vehicle', 'pedestrian', 'cyclist')
        self.tiny = kwargs.get('tiny', False)
        self.tracklet_anno_list, self.tracklet_len_list = self._build_tracklet_anno()
        if self.tiny:
            self.tracklet_anno_list, self.tracklet_len_list = self.tracklet_anno_list[:100], self.tracklet_len_list[:100]
        self.preload_offset = kwargs.get('preload_offset', 10)
        if self.preloading:
            self.training_samples = self._load_data()

    def _build_tracklet_anno(self):
        index = os.path.join(self.Waymo_Folder, f"sot_infos_{self.category_name}_{self.split}.pkl")
        if not os.path.exists(index):
            raise FileNotFoundError(f"{index} not found: run the reference's Waymo conversion (datasets/generate_waymo_sot.py) first")
        with open(index, 'rb') as f:
            infos = pickle.load(f)
        annos = [infos[k] for k in infos.keys()]
        return annos, [len(a) for a in annos]

    def _load_data(self):
        tag = f"{self.split}_{self.category_name}_{self.preload_offset}" + ("_tiny" if self.tiny else "")
        path = os.path.join(self.Waymo_Folder, f"preload_{tag}.dat")
        if os.path.isfile(path):
            with open(path, 'rb') as f:
                return pickle.load(f)
        samples = [[self._get_frame_from_anno(a) for a in annos] for annos in self.tracklet_anno_list]
        with open(path, 'wb') as f:
            pickle.dump(samples, f)
        return samples

    def get_num_tracklets(self):
        return len(self.tracklet_anno_list)

    def get_num_frames_total(self):
        return sum(self.tracklet_len_list)

    def get_num_frames_tracklet(self, tracklet_id):
        return self.tracklet_len_list[tracklet_id]

    def get_frames(self, seq_id, frame_ids):
        if self.preloading:
            return [self.training_samples[seq_id][f] for f in frame_ids]
        annos = self.tracklet_anno_list[seq_id]
        return [self._get_frame_from_anno(annos[f]) for f in frame_ids]

    def tracklets(self):
        return [self.get_frames(i, range(n)) for i, n in enumerate(self.tracklet_len_list)]

    def _get_frame_from_anno(self, anno, track_id=None):
        bb = self.box_from_anno(anno)
        pc = self._global_scan(anno['PC'])
        if self.preload_offset > 0:
            c = bb.corners()
            lo, hi = c.min(1) - self.preload_offset, c.max(1) + self.preload_offset
            pc = PointCloud(pc.points[:, ((pc.points > lo[:, None]) & (pc.points < hi[:, None])).all(0)])
        return {"pc": pc, "3d_bbox": bb, 'meta': anno}

    @staticmethod
    def _pose(lidar_path):
        with open(lidar_path.replace('lidar', 'annos'), 'rb') as f:
            return np.reshape(pickle.load(f)['veh_to_global'], [4, 4]).astype(np.float64)

    @staticmethod
    def _stored_points(lidar_path):
        with open(lidar_path, 'rb') as f:
            return pickle.load(f)['lidars']['points_xyz']

    def _global_scan(self, lidar_path):
        """A frame's whole scan, vehicle -> global (waymo_data.py:121-168)."""
        pts = np.asarray(self._stored_points(lidar_path), dtype=np.float64).T                      # (3, N), vehicle frame
        pose = self._pose(lidar_path)
        R, t = pose[:3, :3], pose[:3, 3]                                                              # veh_pos_to_transform (:170-208)
        return PointCloud((R @ pts + t[:, None]).astype(np.float32))

    def box_from_anno(self, anno):
        """The annotation's box in the global frame."""
        gt = np.array(anno['Box'], dtype=np.float64)
        pose = self._pose(anno['PC'])
        R, t = pose[:3, :3], pose[:3, 3]
        size = [gt[4], gt[3], gt[5]]                                                                  # (l, w, h) -> (w, l, h)
        return Box(R @ gt[0:3] + t, size, R @ _rotz(-gt[-1]))

    # ---- the per-reader interface of the live tracking command line (track.py): scenes, their scans, their raw point rows
    _NAME = re.compile(r"seq_(\d+)_frame_(\d+)\.pkl")

    def _scene_and_frame(self, lidar_path):
        """(scene, frame) of a converter lidar file: from its name `seq_<s>_frame_<f>.pkl`, else from the pickle's scene_name /
        frame_id."""
        m = self._NAME.fullmatch(os.path.basename(lidar_path))
        if m:
            return m.group(1), int(m.group(2))
        with open(lidar_path, 'rb') as f:
            d = pickle.load(f)
        return str(d['scene_name']), int(d['frame_id'])

    def _scan_index(self):
        """{scene: {frame: lidar path}} over the lidar directories the tracklets refer to; the scenes in order of first use."""
        if not hasattr(self, '_scans_of'):
            self._scans_of, self._frame_of = {}, {}
            for annos in self.tracklet_anno_list:
                for a in annos:
                    self._frame_of[a['PC']] = sf = self._scene_and_frame(a['PC'])
                    self._scans_of.setdefault(sf[0], {})
            for d in sorted({os.path.dirname(p) for p in self._frame_of}):
                for name in sorted(os.listdir(d)):
                    if name.endswith('.pkl'):
                        path = os.path.join(d, name)
                        scene, frame = self._frame_of.get(path) or self._scene_and_frame(path)
                        if scene in self._scans_of:
                            self._scans_of[scene][frame] = path
        return self._scans_of

    @property
    def scene_list(self):
        """The scenes the split's tracklets lie in, in order of first appearance."""
        return list(self._scan_index())

    def scene_frames(self, scene):
        """A scene's frame ids, in order."""
        return sorted(self._scan_index().get(scene, {}))

    def anno_frame(self, anno):
        """(scene, frame) of an annotation."""
        self._scan_index()
        return self._frame_of[anno['PC']]

    def scan_size(self, scene, frame):
        """Points in a frame's scan (reads the frame's lidar file)."""
        return len(self._stored_points(self._scan_index()[scene][frame]))

    def raw_scan(self, scene, frame):
        """The scan's rows as stored ((n, 3), float32 or float64) and its one transform, vehicle -> global (3x4)."""
        path = self._scan_index()[scene][frame]
        rows = np.asarray(self._stored_points(path))
        if rows.dtype not in (np.float32, np.float64):
            rows = rows.astype(np.float64)
        return rows.reshape(-1, 3), [self._pose(path)[:3]]

    def read_scan(self, scene, frame):
        """A frame's whole scan in the global frame, as `get_frames` gives it with preload_offset=-1."""
        return self._global_scan(self._scan_index()[scene][frame])
