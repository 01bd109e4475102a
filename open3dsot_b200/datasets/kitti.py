"""KITTI tracking reader with the reference's class and method names (datasets/kitti.py:16-205, base_dataset.py): scene
lists per split, tracklets grouped by `track_id` and ordered by frame, per-frame `{"pc": PointCloud, "3d_bbox": Box,
"meta": anno}` with the box converted from the camera-frame label to the velodyne frame through `Tr_velo_cam`.

Differences in form, not in result: label files are parsed with plain string splitting (no pandas dependency in the data
path), orientations are rotation matrices (`Quaternion(axis=[0,0,-1], radians=a)` is a rotation by -a about +z), and
`tracklets()` hands the whole split to `DeviceTracklets` / `DeviceSiameseSampler` so that batches are then built on the
device.  The directory layout is the reference's: <path>/{velodyne/<scene>/<frame:06>.bin, label_02/<scene>.txt,
calib/<scene>.txt}."""
import os
import pickle
from collections import defaultdict

import numpy as np

from .data_classes import Box, PointCloud

_COLUMNS = ("frame", "track_id", "type", "truncated", "occluded", "alpha", "bbox_left", "bbox_top", "bbox_right", "bbox_bottom",
            "height", "width", "length", "x", "y", "z", "rotation_y")
_KNOWN = ('Car', 'Van', 'Truck', 'Pedestrian', 'Person_sitting', 'Cyclist', 'Tram', 'Misc')


def _rotz(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])


def _rot(axis, a):
    axis = np.asarray(axis, dtype=np.float64) / np.linalg.norm(axis)
    k = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    return np.eye(3) + np.sin(a) * k + (1 - np.cos(a)) * (k @ k)


class BaseDataset:
    def __init__(self, path, split, category_name="Car", **kwargs):
        self.path, self.split, self.category_name = path, split, category_name
        self.preloading = kwargs.get('preloading', False)


class kittiDataset(BaseDataset):
    def __init__(self, path, split, category_name="Car", **kwargs):
        super().__init__(path, split, category_name, **kwargs)
        self.KITTI_Folder = path
        self.KITTI_velo = os.path.join(path, "velodyne")
        self.KITTI_label = os.path.join(path, "label_02")
        self.KITTI_calib = os.path.join(path, "calib")
        self.scene_list = self._build_scene_list(split)
        self.velos = defaultdict(dict)
        self.calibs = {}
        self.coordinate_mode = kwargs.get('coordinate_mode', 'velodyne')
        self.preload_offset = kwargs.get('preload_offset', -1)
        self.tracklet_anno_list, self.tracklet_len_list = self._build_tracklet_anno()
        if self.preloading:
            self.training_samples = self._load_data()

    @staticmethod
    def _build_scene_list(split):
        """kitti.py:33-55: scenes 0-16 train, 17-18 validation, 19-20 test ('tiny' variants: 0 / 18 / 19), else all 21."""
        s = split.upper()
        tiny = "TINY" in s
        if "TRAIN" in s:
            names = [0] if tiny else range(0, 17)
        elif "VALID" in s:
            names = [18] if tiny else range(17, 19)
        elif "TEST" in s:
            names = [19] if tiny else range(19, 21)
        else:
            names = range(21)
        return ['%04d' % n for n in names]

    def _load_data(self):
        path = os.path.join(self.KITTI_Folder,
                            f"preload_kitti_{self.category_name}_{self.split}_{self.coordinate_mode}_{self.preload_offset}.dat")
        if os.path.isfile(path):
            with open(path, 'rb') as f:
                return pickle.load(f)
        samples = [[self._get_frame_from_anno(a) for a in annos] for annos in self.tracklet_anno_list]
        with open(path, 'wb') as f:
            pickle.dump(samples, f)
        return samples

    def get_num_scenes(self):
        return len(self.scene_list)

    def get_num_tracklets(self):
        return len(self.tracklet_anno_list)

    def get_num_frames_total(self):
        return sum(self.tracklet_len_list)

    def get_num_frames_tracklet(self, tracklet_id):
        return self.tracklet_len_list[tracklet_id]

    def _wanted(self, kind):
        c = self.category_name
        if c in _KNOWN:
            return kind == c
        if c == 'All':
            return kind in ('Car', 'Van', 'Pedestrian', 'Cyclist')
        return kind != 'DontCare'

    def _build_tracklet_anno(self):
        """kitti.py:96-133: one list of annotations per (scene, track_id), in order of first appearance, sorted by frame."""
        tracklets, lengths = [], []
        for scene in self.scene_list:
            label_file = os.path.join(self.KITTI_label, scene + ".txt")
            if not os.path.isfile(label_file):
                continue
            per_track = {}
            with open(label_file) as f:
                for line in f:
                    v = line.split()
                    if len(v) < len(_COLUMNS) or not self._wanted(v[2]):
                        continue
                    anno = {"scene": scene}
                    for name, raw in zip(_COLUMNS, v):
                        anno[name] = raw if name == "type" else (int(raw) if name in ("frame", "track_id", "truncated", "occluded")
                                                                 else float(raw))
                    per_track.setdefault(anno["track_id"], []).append(anno)
            for annos in per_track.values():
                annos.sort(key=lambda a: a["frame"])
                tracklets.append(annos)
                lengths.append(len(annos))
        return tracklets, lengths

    def get_frames(self, seq_id, frame_ids):
        if self.preloading:
            return [self.training_samples[seq_id][f] for f in frame_ids]
        annos = self.tracklet_anno_list[seq_id]
        return [self._get_frame_from_anno(annos[f]) for f in frame_ids]

    def tracklets(self):
        """Every tracklet of the split as a list of frames (the input of DeviceTracklets / DeviceSiameseSampler)."""
        return [self.get_frames(i, range(n)) for i, n in enumerate(self.tracklet_len_list)]

    def _get_frame_from_anno(self, anno):
        """kitti.py:144-188."""
        scene_id, frame_id = anno['scene'], anno['frame']
        bb = self.box_from_anno(anno)
        try:
            if frame_id not in self.velos[scene_id]:
                self.velos[scene_id][frame_id] = self._read_scan(scene_id, frame_id)
            pc = self.velos[scene_id][frame_id]
            if self.preload_offset > 0:                       # crop_pc_axis_aligned(pc, bb, offset=preload_offset)
                c = bb.corners()
                lo, hi = c.min(1) - self.preload_offset, c.max(1) + self.preload_offset
                keep = ((pc.points > lo[:, None]) & (pc.points < hi[:, None])).all(0)
                pc = PointCloud(pc.points[:, keep])
        except (OSError, ValueError):
            pc = PointCloud(np.array([[0, 0, 0]], dtype=np.float32).T)
        return {"pc": pc, "3d_bbox": bb, 'meta': anno}

    def _velo_to_cam(self, scene_id):
        if scene_id not in self.calibs:
            self.calibs[scene_id] = self._read_calib_file(os.path.join(self.KITTI_calib, scene_id + ".txt"))
        return np.vstack((self.calibs[scene_id]["Tr_velo_cam"], np.array([0, 0, 0, 1])))

    def box_from_anno(self, anno):
        """The label's box in the reader's coordinate_mode (kitti.py:150-163), without loading the scan."""
        velo_to_cam = self._velo_to_cam(anno['scene'])
        size = [anno["width"], anno["length"], anno["height"]]
        if self.coordinate_mode == 'velodyne':
            center_cam = np.array([anno["x"], anno["y"] - anno["height"] / 2, anno["z"], 1])
            center = (np.linalg.inv(velo_to_cam) @ center_cam)[:3]
            rot = _rotz(-anno["rotation_y"]) @ _rotz(-np.pi / 2)
        else:
            center = [anno["x"], anno["y"] - anno["height"] / 2, anno["z"]]
            rot = _rot([0, 1, 0], anno["rotation_y"]) @ _rot([1, 0, 0], np.pi / 2)
        return Box(center, size, rot)

    def _read_scan(self, scene_id, frame_id):
        pts = np.fromfile(self.scan_path(scene_id, frame_id), dtype=np.float32).reshape(-1, 4).T
        pc = PointCloud(pts)
        if self.coordinate_mode == "camera":
            pc.points = (self._velo_to_cam(scene_id) @ np.vstack((pc.points[:3], np.ones(pc.points.shape[1]))))[:3]
        return pc

    def scan_path(self, scene_id, frame_id):
        return os.path.join(self.KITTI_velo, scene_id, '{:06}.bin'.format(frame_id))

    # ---- the per-reader interface of the live tracking command line (track.py): scenes, their scans, their raw point rows
    def scene_frames(self, scene_id):
        """The frame numbers of a scene's scans, in order: 0 .. its last velodyne file or labelled frame."""
        d = os.path.join(self.KITTI_velo, scene_id)
        names = os.listdir(d) if os.path.isdir(d) else []
        last = max((int(n[:-4]) for n in names if n.endswith(".bin") and n[:-4].isdigit()), default=-1)
        for annos in self.tracklet_anno_list:
            if annos[0]["scene"] == scene_id:
                last = max(last, annos[-1]["frame"])
        return list(range(last + 1))

    @staticmethod
    def anno_frame(anno):
        """(scene, frame) of an annotation."""
        return anno["scene"], anno["frame"]

    def scan_size(self, scene_id, frame_id):
        """Points in a frame's scan, from the file size (16 bytes per point; 1 for the placeholder of a missing file)."""
        path = self.scan_path(scene_id, frame_id)
        return max(os.path.getsize(path) // 16, 1) if os.path.isfile(path) else 1

    def raw_scan(self, scene_id, frame_id):
        """The scan's rows as stored ((n, 4) float32: x, y, z, reflectance) and the transforms `read_scan` applies to them:
        none in velodyne mode, Tr_velo_cam (3x4) in camera mode.  A missing or unreadable file gives the placeholder point."""
        try:
            rows = np.fromfile(self.scan_path(scene_id, frame_id), dtype=np.float32).reshape(-1, 4)
            return rows, ([self._velo_to_cam(scene_id)[:3]] if self.coordinate_mode == "camera" else [])
        except (OSError, ValueError):
            return np.zeros((1, 3), np.float32), []

    def read_scan(self, scene_id, frame_id):
        """The whole scan of a frame in the reader's coordinate_mode, not cached and not cropped (a missing or unreadable
        file gives the reader's one-point placeholder)."""
        try:
            return self._read_scan(scene_id, frame_id)
        except (OSError, ValueError):
            return PointCloud(np.array([[0, 0, 0]], dtype=np.float32).T)

    @staticmethod
    def _read_calib_file(filepath):
        """kitti.py:190-205: every line that parses as twelve floats becomes a 3x4 matrix keyed by its first token."""
        data = {}
        with open(filepath) as f:
            for line in f:
                v = line.split()
                try:
                    data[v[0]] = np.array([float(x) for x in v[1:]]).reshape(3, 4)
                except (ValueError, IndexError):
                    pass
        return data
