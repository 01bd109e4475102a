"""Compact stand-ins for the reference's shipped Lightning checkpoints, for tests/test_checkpoint_compat.py.

Each fixture is the reference's own `pretrained_models/<name>.ckpt` (pytorch-lightning 1.3.8, legacy non-zip torch format)
read with the package's restricted unpickler and written back in the same legacy format (pickle protocol 4 instead of 2,
for size) with the same top-level keys, state-dict names, order, shapes and dtypes, scheduler / callback entries and
`easydict.EasyDict` hyper-parameters.  What is left out is the bulk: every tensor is a view of one shared single-element
storage of its dtype (value 1, stride 0), and the optimizer's per-parameter Adam moments are dropped
(`optimizer_states[i]["state"]` empty, its param_groups kept), so a file is about 20 KB instead of 17-27 MB.
Regenerate with  python tests/golden/make_ckpt_fixtures.py <reference checkout>/pretrained_models
"""
import os
import sys
import types

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from open3dsot_b200.checkpoint import load_lightning_checkpoint  # noqa: E402
from open3dsot_b200.compat import easydict as _ed  # noqa: E402

NAMES = ("bat_kitti_car", "bat_kitti_pedestrian", "mmtrack_kitti_car")


_ONE = {}   # one single-element storage per dtype, shared by every tensor of that dtype


def shrink(obj):
    if isinstance(obj, torch.Tensor):
        if obj.dim() == 0 or obj.numel() == 0:
            return obj.clone()
        return _ONE.setdefault(obj.dtype, torch.ones(1, dtype=obj.dtype)).expand(obj.shape)
    if isinstance(obj, dict):
        out = type(obj)() if type(obj) is not dict else {}
        for k, v in obj.items():
            out[k] = shrink(v)
        return out
    if isinstance(obj, list):
        return [shrink(v) for v in obj]
    if isinstance(obj, tuple):
        return tuple(shrink(v) for v in obj)
    return obj


def classes_in(obj, acc):
    if isinstance(obj, dict):
        for k, v in obj.items():
            classes_in(k, acc)
            classes_in(v, acc)
    elif isinstance(obj, (list, tuple)):
        for v in obj:
            classes_in(v, acc)
    elif isinstance(obj, type):
        acc.add(obj)
    elif not isinstance(obj, (torch.Tensor, str, bytes, int, float, bool, type(None))) and type(obj).__module__ != "builtins":
        acc.add(type(obj))
        classes_in(getattr(obj, "__dict__", {}), acc)
    return acc


def write(ck, path):
    """torch.save in the legacy format, every class under the module / name the reference environment resolves it by."""
    saved = dict(sys.modules)
    ed = _ed.EasyDict
    old_ed = (ed.__module__, ed.__qualname__)
    try:
        ed.__module__, ed.__qualname__ = "easydict", "EasyDict"
        for cls in classes_in(ck, set()) | {ed}:
            parts = cls.__module__.split(".")
            for i in range(1, len(parts) + 1):
                sys.modules.setdefault(".".join(parts[:i]), types.ModuleType(".".join(parts[:i])))
            setattr(sys.modules[cls.__module__], cls.__qualname__, cls)
        torch.save(ck, path, _use_new_zipfile_serialization=False, pickle_protocol=4)
    finally:
        ed.__module__, ed.__qualname__ = old_ed
        sys.modules.clear()
        sys.modules.update(saved)


def main(src_dir):
    os.makedirs(os.path.join(HERE, "ckpt"), exist_ok=True)
    for name in NAMES:
        ck = load_lightning_checkpoint(os.path.join(src_dir, name + ".ckpt"))
        for opt in ck.get("optimizer_states", []):
            if isinstance(opt, dict) and "state" in opt:
                opt["state"] = {}
        out = os.path.join(HERE, "ckpt", name + ".ckpt")
        write(shrink(ck), out)
        print(out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main(sys.argv[1])
