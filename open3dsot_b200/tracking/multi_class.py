"""Live tracking of several object classes over shared scan feeds: one model per class, one scan ingest, one step per class.

Every class keeps its own model, config, weights and static-weight caches, and its own `MultiTargetTracker` (its slots, its
`max_targets`, its template mode, its motion or siamese inputs, its occupancy buckets and their captured steps), all built over
one `ScanFeeds` store.  `advance()` brings the staged scans in once (one packed host->device copy and one `o3d_scan_ingest`
launch for every feed), then every class picks the bucket of its own work list and replays that bucket's captured step on its
own side stream, forked from the current stream before and joined into it after, the fork / join `fused.run_ahead` uses for the
template and search branches.  A class with nothing to advance replays nothing.  Each class's bucket graphs share one memory
pool, and the classes keep separate pools, since they replay side by side.  The classes may be different model families (BAT
for cars, M2-Track for pedestrians).

A target is named (class, id); ids are unique within a class and key the target's draws as in a lone tracker, so its boxes
depend neither on the other classes nor on their slot counts: they are bitwise what a `MultiTargetTracker` of its class with
the same seed, scans and add / drop schedule gives it.  The classes must agree on the frame conventions their boxes and metrics
are read in (`up_axis`, `IoU_space`, `degrees`)."""
import torch

from .. import runtime
import numpy as np

from .multi_tracker import (MultiTargetTracker, ScanFeeds, check_births, check_coast, check_detections, check_lost_rule,
                            class_peaks, feed_schedule, refuse_births, run_scenes)

SHARED_KEYS = ("up_axis", "IoU_space", "degrees")


class MultiClassTracker:
    """`models` {class name: model}, `max_targets` {class name: slots}, over `feeds` scan feeds (a number, or a `ScanFeeds`
    store) of at most `max_points` points per scan.  `seed`, `use_graph` and `precision` as for MultiTargetTracker, for every
    class; `lost` is one end-of-track rule for every class (MultiTargetTracker's `lost=`) or {class: rule}, a class without an
    entry never losing a target; `coast` likewise one alpha (MultiTargetTracker's `coast=`) or {class: alpha}, a class without
    an entry never coasting (a class that coasts needs a rule); `detections` likewise one (max_per_scan, gate) or
    {class: (max_per_scan, gate)}, a class without an entry taking no detections; `births` likewise one (min_score, per_scan) or
    {class: (min_score, per_scan)}, a class without an entry starting no target itself (a class with births needs detections),
    and `births()` returns {class: MultiTargetTracker.births()} of those classes.  `put` / `put_raw` / `advance()` as on
    MultiTargetTracker, with a scan's detections given per class ({class: rows}); `add(cls, id, box, feed=)` / `drop(cls, id)`
    start and end a target of a class."""

    def __init__(self, models, max_points, max_targets, feeds=1, seed=0, use_graph=True, precision="fp32", lost=None, coast=None,
                 detections=None, births=None):
        if not models:
            raise ValueError("MultiClassTracker: no classes; give one model per class")
        self.precision = runtime.check_precision(precision)
        names = list(models)
        for n in names:
            if n not in max_targets:
                raise ValueError(f"max_targets: class {n!r} has no slot count")
        for n in max_targets:
            if n not in models:
                raise ValueError(f"max_targets: class {n!r} has no model")
        rules = lost if isinstance(lost, dict) else {n: lost for n in names}
        for n in rules:
            if n not in models:
                raise ValueError(f"lost: class {n!r} has no model")
        rules = {n: check_lost_rule(rules.get(n)) for n in names}
        coasts = coast if isinstance(coast, dict) else {n: coast for n in names}
        for n in coasts:
            if n not in models:
                raise ValueError(f"coast: class {n!r} has no model")
        for n in names:
            try:
                coasts[n] = check_coast(coasts.get(n), rules[n])
            except ValueError as e:
                raise ValueError(f"class {n!r}: {e}") from None
        dets = detections if isinstance(detections, dict) else {n: detections for n in names}
        for n in dets:
            if n not in models:
                raise ValueError(f"detections: class {n!r} has no model")
        for n in names:
            try:
                dets[n] = check_detections(dets.get(n))
            except ValueError as e:
                raise ValueError(f"class {n!r}: {e}") from None
        born = births if isinstance(births, dict) else {n: births for n in names}
        for n in born:
            if n not in models:
                raise ValueError(f"births: class {n!r} has no model")
        for n in names:
            try:
                born[n] = check_births(born.get(n), dets[n])
            except ValueError as e:
                raise ValueError(f"class {n!r}: {e}") from None
        c0 = models[names[0]].config
        for n in names[1:]:
            c = models[n].config
            for key in SHARED_KEYS:
                a, b = c0.get(key), c.get(key)
                if (list(a) if isinstance(a, (list, tuple)) else a) != (list(b) if isinstance(b, (list, tuple)) else b):
                    raise ValueError(f"class {n!r}: {key}={b} differs from class {names[0]!r}'s {key}={a}; the classes of one "
                                     f"tracker share the frame their boxes are read in")
        self.dev = dev = next(models[names[0]].parameters()).device
        self.scan_feeds = feeds if isinstance(feeds, ScanFeeds) else ScanFeeds(max_points, feeds, dev)
        self.scan_feeds.claim(self)                       # before the class trackers: they share the store, this one advances it
        self.F = self.scan_feeds.F
        self.trackers = {}
        for n in names:
            try:
                self.trackers[n] = MultiTargetTracker(models[n], max_points, max_targets[n], seed=seed, use_graph=use_graph,
                                                      feeds=self.scan_feeds, precision=precision, lost=rules[n], coast=coasts[n],
                                                      detections=dets[n], births=born[n])
            except ValueError as e:
                self.scan_feeds.owner = None
                raise ValueError(f"class {n!r}: {e}") from None
        # row offset of every class's slots in snapshot()
        self.offset, k = {}, 0
        for n, trk in self.trackers.items():
            self.offset[n], k = k, k + trk.K
        self.K = k
        self._streams = {n: torch.cuda.Stream(device=dev) for n in names} if dev.type == "cuda" else {}

    # ------------------------------------------------------------------ one step: every class's bucket step on its own stream
    def _run(self, fed):
        if not self._streams:
            for trk in self.trackers.values():
                trk._run(fed)
            return
        cur = torch.cuda.current_stream()
        for n, trk in self.trackers.items():
            side = self._streams[n]
            side.wait_stream(cur)
            with torch.cuda.stream(side):
                trk._run(fed)
        for side in self._streams.values():
            cur.wait_stream(side)

    # ------------------------------------------------------------------ public interface
    def _class(self, cls):
        trk = self.trackers.get(cls)
        if trk is None:
            raise ValueError(f"class {cls!r} is not tracked here; the classes are {list(self.trackers)}")
        return trk

    def _check_detections(self, feed, detections):
        """A put's {class: rows}, each checked by its class tracker (ValueError) before anything is staged."""
        if detections is None:
            return {}
        if not isinstance(detections, dict):
            raise ValueError("detections: expected {class: (M, 16) rows}")
        out = {}
        for n, rows in detections.items():
            try:
                out[n] = self._class(n)._check_detections(feed, rows)
            except ValueError as e:
                raise ValueError(f"class {n!r}: {e}") from None
        return out

    def put(self, feed, points, n_valid=None, detections=None):
        """Stage the next scan of `feed` for every class (ScanFeeds.put), with its detections per class ({class: rows}, for the
        classes built with detections=).  No host sync."""
        rows = self._check_detections(feed, detections)
        self.scan_feeds.put(feed, points, n_valid)
        for n, r in rows.items():
            self.trackers[n]._stage_detections(feed, r)

    def put_raw(self, feed, rows, transforms=(), detections=None):
        """Stage the next scan of `feed` as a reader stores it (ScanFeeds.put_raw); the next `advance()` ingests it.  `detections`
        as for `put`."""
        det = self._check_detections(feed, detections)
        self.scan_feeds.put_raw(feed, rows, transforms)
        for n, r in det.items():
            self.trackers[n]._stage_detections(feed, r)

    def advance(self):
        """Bring in every staged scan (one copy, one ingest) and advance every class's active targets of those feeds to it, each
        class in one replay of its bucket's captured step.  Returns {class: that class tracker's boxes()}, device views; no host sync."""
        fed = set(self.scan_feeds.staged)
        self.scan_feeds.ingest()
        self._run(fed)
        return {n: trk.boxes() for n, trk in self.trackers.items()}

    def step(self, points, n_valid=None):
        """One-feed form: `put(0, points)` + `advance()`."""
        if self.F != 1:
            raise ValueError(f"step() drives a one-feed tracker; with feeds={self.F} use put() / put_raw() and advance()")
        self.put(0, points, n_valid)
        return self.advance()

    def add(self, cls, target_id, box, feed=0):
        """Start target `target_id` of class `cls` on the most recent scan of `feed` with `box` (MultiTargetTracker.add)."""
        self._class(cls).add(target_id, box, feed=feed)

    def drop(self, cls, target_id):
        """End target `target_id` of class `cls` and free its slot."""
        self._class(cls).drop(target_id)

    def targets(self):
        """{(class, target id): row of snapshot()} of the active targets (host state)."""
        return {(n, tid): self.offset[n] + k for n, trk in self.trackers.items() for tid, k in trk.slot_of.items()}

    def snapshot(self):
        """A device copy of every class's slots, (sum of max_targets, 15), the classes in order: MultiTargetTracker.snapshot's
        rows of each."""
        return torch.cat([trk.snapshot() for trk in self.trackers.values()])

    def evidence(self):
        """Every class's MultiTargetTracker.evidence() rows, (sum of max_targets, 4), the rows of snapshot()."""
        return torch.cat([trk.evidence() for trk in self.trackers.values()])

    def _record(self):
        return torch.cat([trk._record() for trk in self.trackers.values()])

    def _coast_rows(self):
        return np.concatenate([trk._coast_rows() for trk in self.trackers.values()])

    def _match_record(self):
        return torch.cat([trk._match_record() for trk in self.trackers.values()])

    def _detect_rows(self):
        return np.concatenate([trk._detect_rows() for trk in self.trackers.values()])

    def unmatched(self):
        """{class: {feed: [(index, data_classes.Box, score), ...]}}: MultiTargetTracker.unmatched() of every class built with
        detections=, read back from the device together (one sync)."""
        classes = [n for n, trk in self.trackers.items() if trk.detections is not None]
        if not classes:
            raise ValueError("unmatched(): no class was built with detections=")
        flats = [self.trackers[n]._unmatched_device() for n in classes]
        host = torch.cat(flats).cpu().numpy()
        out, at = {}, 0
        for n, flat in zip(classes, flats):
            out[n] = self.trackers[n]._unmatched_decode(host[at:at + flat.numel()])
            at += flat.numel()
        return out

    def births(self, wait=False):
        """{class: [(id, feed, slot, detection index), ...]}: MultiTargetTracker.births(wait) of every class built with births=."""
        classes = [n for n, trk in self.trackers.items() if trk.birth_rule is not None]
        if not classes:
            raise ValueError("births(): no class was built with births=")
        return {n: self.trackers[n].births(wait) for n in classes}

    def lost_targets(self):
        """(class, id) of the active targets their class's rule has declared lost, read back from the device (one sync)."""
        lost = torch.cat([trk.lost for trk in self.trackers.values()]).cpu().numpy()
        return sorted(key for key, k in self.targets().items() if lost[k])

    def drop_lost(self):
        """`drop` every target of `lost_targets()`; returns their (class, id)."""
        keys = self.lost_targets()
        for key in keys:
            self.drop(*key)
        return keys

    def results(self):
        """{(class, target id): data_classes.Box} of the active targets, read back from the device once."""
        from ..datasets.data_classes import Box
        host = self.snapshot().cpu().double().numpy()
        return {key: Box(host[k, 0:3], host[k, 3:6], host[k, 6:15].reshape(3, 3)) for key, k in self.targets().items()}


def track_classes(models, scenes, feeds, max_targets, seed=0, max_points=None, use_graph=True, chunk=256, precision="fp32",
                  lost=None, evidence=False, coast=None, detections=None, births=None):
    """`track_feeds` for several classes through one MultiClassTracker.  `models` and `max_targets`: {class: model},
    {class: slots}.  A scene's targets are named (class, id): "starts": {t: [((class, id), Box), ...]}, "ends": {(class, id):
    last t}; (class, id) is unique over all scenes.  A scene is admitted when a feed is free and every class has the scene's
    peak of that class free.  Returns, per scene, {(class, id): {t: data_classes.Box}}.  `lost`: one end-of-track rule or
    {class: rule} (MultiClassTracker); a lost target's results end at the frame it was declared lost on.  With `evidence`, also
    returns, per scene, {(class, id): {t: (points in the box, score)}}, with a third value, whether the frame was coasted, for
    the classes that coast (`coast`: one alpha or {class: alpha}, MultiClassTracker).  `detections`: one (max_per_scan, gate) or
    {class: (max_per_scan, gate)} (MultiClassTracker); a scene's "detections": t -> {class: rows} of its scan t, and the
    evidence of the classes that take detections ends with (reacquired, detection) (run_scenes).  `births` is refused, as by
    track_feeds."""
    refuse_births(births, "track_classes")
    runtime.check_precision(precision)
    if max_points is None:
        raise ValueError("track_classes: give max_points, the largest scan of the scenes")
    lengths = [int(sc["frames"]) for sc in scenes]
    for i, sc in enumerate(scenes):
        for group in sc["starts"].values():
            for key, _ in group:
                if key[0] not in models:
                    raise ValueError(f"scene {i}: target {key} is of class {key[0]!r}, which has no model")
    peaks = [class_peaks(lengths[i], sc["starts"], sc["ends"]) for i, sc in enumerate(scenes)]
    sched = feed_schedule(lengths, peaks, feeds, max_targets)
    trk = MultiClassTracker(models, max_points, max_targets, feeds=feeds, seed=seed, use_graph=use_graph, precision=precision,
                            lost=lost, coast=coast, detections=detections)
    return run_scenes(trk, lambda key, box, f: trk.add(*key, box, feed=f), lambda key: trk.drop(*key), scenes, sched, chunk,
                      evidence)
