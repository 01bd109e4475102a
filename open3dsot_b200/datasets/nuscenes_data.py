"""nuScenes reader with the reference's class and method names (datasets/nuscenes_data.py:59-173) — WITHOUT nuscenes-devkit:
the dataset's JSON tables (<path>/<version>/{scene, sample, sample_data, sample_annotation, instance, category, ego_pose,
calibrated_sensor, sensor}.json) are read directly and indexed the way the devkit's `NuScenes.__init__` does
(`sample['data'][channel]` for key-frame sample_data records, `sample_annotation['category_name']` through its instance),
LiDAR sweeps are the devkit's `.pcd.bin` layout (float32 x, y, z, intensity, ring index), and quaternions are turned into
rotation matrices by `quat_to_rot` (w, x, y, z).  A frame is `{"pc": PointCloud, "3d_bbox": Box, "meta": anno}` with the cloud
moved sensor -> ego -> global (nuscenes_data.py:155-168) and the box as annotated in the global frame.

Scene splits.  The devkit's `create_splits_scenes()` is a hard-coded list of scene names per split; it is not reproduced
here.  In order of precedence: `scenes=[...]` keyword, a file `<path>/splits/<split>.txt` (one scene name per line), the two
v1.0-mini splits (known), the devkit itself when it happens to be installed; otherwise a ValueError that says so."""
import json
import os
import pickle

import numpy as np

from .data_classes import Box, PointCloud
from .kitti import BaseDataset

tracking_to_general_class = {
    'void / ignore': ['animal', 'human.pedestrian.personal_mobility', 'human.pedestrian.stroller', 'human.pedestrian.wheelchair',
                      'movable_object.barrier', 'movable_object.debris', 'movable_object.pushable_pullable', 'movable_object.trafficcone',
                      'static_object.bicycle_rack', 'vehicle.emergency.ambulance', 'vehicle.emergency.police', 'vehicle.construction'],
    'bicycle': ['vehicle.bicycle'], 'bus': ['vehicle.bus.bendy', 'vehicle.bus.rigid'], 'car': ['vehicle.car'],
    'motorcycle': ['vehicle.motorcycle'],
    'pedestrian': ['human.pedestrian.adult', 'human.pedestrian.child', 'human.pedestrian.construction_worker', 'human.pedestrian.police_officer'],
    'trailer': ['vehicle.trailer'], 'truck': ['vehicle.truck']}
general_to_tracking_class = {g: t for t, gs in tracking_to_general_class.items() for g in gs}

_MINI = {"mini_train": ["scene-0061", "scene-0553", "scene-0655", "scene-0757", "scene-0796", "scene-1077", "scene-1094", "scene-1100"],
         "mini_val": ["scene-0103", "scene-0916"]}


def quat_to_rot(q):
    """(w, x, y, z) -> 3x3 rotation matrix (pyquaternion `Quaternion(q).rotation_matrix`)."""
    w, x, y, z = np.asarray(q, dtype=np.float64) / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


class _Tables:
    """The devkit's token-indexed tables plus its two reverse indices."""
    NAMES = ("scene", "sample", "sample_data", "sample_annotation", "instance", "category", "ego_pose", "calibrated_sensor", "sensor")

    def __init__(self, root):
        self.t = {}
        for n in self.NAMES:
            with open(os.path.join(root, n + ".json")) as f:
                self.t[n] = json.load(f)
        self.by = {n: {r["token"]: r for r in rows} for n, rows in self.t.items()}
        for r in self.t["sample"]:
            r["data"] = {}
        for sd in self.t["sample_data"]:                      # NuScenes.__make_reverse_index__: key-frame data per channel
            if sd["is_key_frame"]:
                cs = self.by["calibrated_sensor"][sd["calibrated_sensor_token"]]
                self.by["sample"][sd["sample_token"]]["data"][self.by["sensor"][cs["sensor_token"]]["channel"]] = sd["token"]
        for a in self.t["sample_annotation"]:
            inst = self.by["instance"][a["instance_token"]]
            a["category_name"] = self.by["category"][inst["category_token"]]["name"]

    def get(self, table, token):
        return self.by[table][token]


class NuScenesDataset(BaseDataset):
    def __init__(self, path, split, category_name="Car", version='v1.0-trainval', **kwargs):
        super().__init__(path, split, category_name, **kwargs)
        self.nusc = _Tables(os.path.join(path, version))
        self.version = version
        self.key_frame_only = kwargs.get('key_frame_only', False)
        self.min_points = kwargs.get('min_points', False)
        self.preload_offset = kwargs.get('preload_offset', -1)
        self._scenes = self._split_scenes(split, kwargs.get('scenes'))
        self.track_instances = self.filter_instance(split, category_name.lower(), self.min_points)
        self.tracklet_anno_list, self.tracklet_len_list = self._build_tracklet_anno()
        if self.preloading:
            self.training_samples = self._load_data()

    def _split_scenes(self, split, scenes):
        if scenes is not None:
            return set(scenes)
        f = os.path.join(self.path, "splits", f"{split}.txt")
        if os.path.isfile(f):
            with open(f) as fh:
                return {line.strip() for line in fh if line.strip()}
        if split in _MINI:
            return set(_MINI[split])
        try:
            from nuscenes.utils.splits import create_splits_scenes     # only when the devkit is installed
            return set(create_splits_scenes()[split])
        except Exception:
            raise ValueError(f"nuScenes split '{split}': give scenes=[...], or write {f} (one scene name per line); the devkit's "
                             "hard-coded split lists are not part of this package")

    def filter_instance(self, split, category_name=None, min_points=-1):
        """nuscenes_data.py:72-92: instances whose first annotation lies in a scene of the split, has >= min_points LiDAR points
        and (when a tracking class is given) one of its general categories."""
        general = tracking_to_general_class[category_name] if category_name is not None else None
        out = []
        for inst in self.nusc.t["instance"]:
            anno = self.nusc.get('sample_annotation', inst['first_annotation_token'])
            sample = self.nusc.get('sample', anno['sample_token'])
            scene = self.nusc.get('scene', sample['scene_token'])
            cat = self.nusc.get('category', inst['category_token'])['name']
            if scene['name'] in self._scenes and anno['num_lidar_pts'] >= min_points and (general is None or cat in general):
                out.append(inst)
        return out

    def _build_tracklet_anno(self):
        """nuscenes_data.py:94-115: follow each instance's annotation chain (`next`), optionally key frames only."""
        tracklets, lengths = [], []
        for inst in self.track_instances:
            track, token = [], inst['first_annotation_token']
            while token != '':
                ann = self.nusc.get('sample_annotation', token)
                sample = self.nusc.get('sample', ann['sample_token'])
                sd = self.nusc.get('sample_data', sample['data']['LIDAR_TOP'])
                token = ann['next']
                if self.key_frame_only and not sd['is_key_frame']:
                    continue
                track.append({"sample_data_lidar": sd, "box_anno": ann})
            tracklets.append(track)
            lengths.append(len(track))
        return tracklets, lengths

    def _load_data(self):
        path = os.path.join(self.path, f"preload_nuscenes_{self.category_name}_{self.split}_{self.version}_{self.preload_offset}_{self.min_points}.dat")
        if os.path.isfile(path):
            with open(path, 'rb') as f:
                return pickle.load(f)
        samples = [[self._get_frame_from_anno_data(a) for a in annos] for annos in self.tracklet_anno_list]
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
        return [self._get_frame_from_anno_data(annos[f]) for f in frame_ids]

    def tracklets(self):
        return [self.get_frames(i, range(n)) for i, n in enumerate(self.tracklet_len_list)]

    def _get_frame_from_anno_data(self, anno):
        """nuscenes_data.py:152-173."""
        bb = self.box_from_anno(anno)
        pc = self._global_scan(anno['sample_data_lidar'])
        if self.preload_offset > 0:                               # crop_pc_axis_aligned(pc, bb, offset=preload_offset)
            c = bb.corners()
            lo, hi = c.min(1) - self.preload_offset, c.max(1) + self.preload_offset
            pc = PointCloud(pc.points[:, ((pc.points > lo[:, None]) & (pc.points < hi[:, None])).all(0)])
        return {"pc": pc, "3d_bbox": bb, 'meta': anno}

    def _global_scan(self, sd):
        """A LiDAR sample_data's whole scan, sensor -> ego -> global (nuscenes_data.py:159-167)."""
        scan = np.fromfile(os.path.join(self.path, sd['filename']), dtype=np.float32).reshape(-1, 5)[:, :3].T.astype(np.float64)
        cs = self.nusc.get('calibrated_sensor', sd['calibrated_sensor_token'])
        scan = quat_to_rot(cs['rotation']) @ scan + np.array(cs['translation'])[:, None]                 # sensor -> ego
        pose = self.nusc.get('ego_pose', sd['ego_pose_token'])
        scan = quat_to_rot(pose['rotation']) @ scan + np.array(pose['translation'])[:, None]             # ego -> global
        return PointCloud(scan.astype(np.float32))

    @staticmethod
    def box_from_anno(anno):
        """The annotation's box, as annotated in the global frame."""
        box_anno = anno['box_anno']
        return Box(box_anno['translation'], box_anno['size'], quat_to_rot(box_anno['rotation']))

    # ---- the per-reader interface of the live tracking command line (track.py): scenes, their scans, their raw point rows
    @property
    def scene_list(self):
        """The split's scenes, in the scene table's order."""
        return [s['name'] for s in self.nusc.t['scene'] if s['name'] in self._scenes]

    def _scene_scans(self, scene):
        """A scene's key-frame LIDAR_TOP sample_data records in timestamp order (the only scans the tracklets refer to)."""
        if not hasattr(self, '_scans_of'):
            self._scans_of = {}
            token_of = {s['token']: s['name'] for s in self.nusc.t['scene']}
            for smp in self.nusc.t['sample']:
                if 'LIDAR_TOP' in smp['data']:
                    self._scans_of.setdefault(token_of[smp['scene_token']], []).append(
                        self.nusc.get('sample_data', smp['data']['LIDAR_TOP']))
            for sds in self._scans_of.values():
                sds.sort(key=lambda sd: sd['timestamp'])
            self._frame_of = {sd['token']: i for sds in self._scans_of.values() for i, sd in enumerate(sds)}
        return self._scans_of.get(scene, [])

    def scene_frames(self, scene):
        """A scene's frames: the positions 0 .. n-1 of its key-frame scans in timestamp order."""
        return list(range(len(self._scene_scans(scene))))

    def anno_frame(self, anno):
        """(scene, frame) of an annotation."""
        sd = anno['sample_data_lidar']
        scene = self.nusc.get('scene', self.nusc.get('sample', sd['sample_token'])['scene_token'])['name']
        self._scene_scans(scene)
        return scene, self._frame_of[sd['token']]

    def scan_size(self, scene, frame):
        """Points in a frame's scan, from the file size (20 bytes per point)."""
        return os.path.getsize(os.path.join(self.path, self._scene_scans(scene)[frame]['filename'])) // 20

    def raw_scan(self, scene, frame):
        """The scan's rows as stored ((n, 5) float32) and its two transforms, sensor -> ego then ego -> global (3x4 each)."""
        sd = self._scene_scans(scene)[frame]
        rows = np.fromfile(os.path.join(self.path, sd['filename']), dtype=np.float32).reshape(-1, 5)
        cs = self.nusc.get('calibrated_sensor', sd['calibrated_sensor_token'])
        pose = self.nusc.get('ego_pose', sd['ego_pose_token'])
        return rows, [np.hstack([quat_to_rot(r['rotation']), np.array(r['translation'], np.float64)[:, None]]) for r in (cs, pose)]

    def read_scan(self, scene, frame):
        """A frame's whole scan in the global frame, as `get_frames` gives it with preload_offset=-1."""
        return self._global_scan(self._scene_scans(scene)[frame])
