"""Reading the reference's Lightning checkpoints (`pretrained_models/*.ckpt`, written by pytorch-lightning 1.3.8 in the
legacy non-zip torch format) without pytorch_lightning / easydict installed.

Such a file pickles, besides tensors, an `easydict.EasyDict` (hyper_parameters.config) and a
`pytorch_lightning.callbacks.model_checkpoint.ModelCheckpoint` class used as a dict key (SURVEY.md §2.1 row 19, §5).
`load_lightning_checkpoint` unpickles with a restricted `find_class`: only an explicit whitelist of (module, name)
pairs resolves to the real object — the tensor / storage rebuild helpers, `collections.OrderedDict`, the numpy array /
scalar reconstruction helpers and a few inert builtins containers; `easydict.EasyDict` maps to our stand-in; EVERY other
global (including `builtins.eval/exec/getattr/__import__`, `os.*`, `torch.hub.*`, `numpy.testing.*`) becomes an inert
placeholder class whose construction and `__setstate__` do nothing, so a crafted file cannot call into them.  The result has
the reference's keys: `state_dict`, `hyper_parameters`, `epoch`, `global_step`, `optimizer_states`, …
"""
import pickle

import torch

from .compat.easydict import EasyDict

_STORAGES = {n for n in ("DoubleStorage", "FloatStorage", "HalfStorage", "BFloat16Storage", "LongStorage", "IntStorage",
                        "ShortStorage", "CharStorage", "ByteStorage", "BoolStorage", "UntypedStorage")}
# exact (module, name) pairs that resolve to the real object; nothing else does
_SAFE = {
    ("collections", "OrderedDict"), ("collections", "defaultdict"),
    ("torch._utils", "_rebuild_tensor_v2"), ("torch._utils", "_rebuild_tensor"), ("torch._utils", "_rebuild_parameter"),
    ("torch", "Size"), ("torch", "device"), ("torch", "dtype"),
    ("torch.serialization", "_get_layout"),
    ("numpy.core.multiarray", "_reconstruct"), ("numpy.core.multiarray", "scalar"),
    ("numpy._core.multiarray", "_reconstruct"), ("numpy._core.multiarray", "scalar"),
    ("numpy", "ndarray"), ("numpy", "dtype"),
    ("_codecs", "encode"),
    ("builtins", "set"), ("builtins", "frozenset"), ("builtins", "slice"), ("builtins", "complex"),
    ("builtins", "bytearray"), ("builtins", "list"), ("builtins", "dict"), ("builtins", "tuple"),
    ("builtins", "int"), ("builtins", "float"), ("builtins", "bool"), ("builtins", "str"), ("builtins", "bytes"),
} | {("torch", n) for n in _STORAGES} | {("torch.storage", "UntypedStorage"), ("torch.storage", "TypedStorage")}


def _placeholder(module, name):
    return type(name, (), {"__module__": module, "__init__": lambda self, *a, **k: None,
                           "__setstate__": lambda self, state: None, "__reduce__": lambda self: (str, ("",))})


class _RestrictedUnpickler(pickle.Unpickler):
    def find_class(self, module, name):
        if module == "easydict" and name == "EasyDict":
            return EasyDict
        if (module, name) in _SAFE:
            return super().find_class(module, name)
        if module == "torch" and name.endswith("dtype"):
            return super().find_class(module, name)
        return _placeholder(module, name)


class _PickleModule:
    """The `pickle_module` torch.load expects: module-like object exposing Unpickler / load / loads."""
    __name__ = "open3dsot_b200_restricted_pickle"
    Unpickler = _RestrictedUnpickler
    Pickler = pickle.Pickler
    PickleError = pickle.PickleError
    UnpicklingError = pickle.UnpicklingError

    @staticmethod
    def load(f, **kw):
        return _RestrictedUnpickler(f, **kw).load()

    @staticmethod
    def loads(b, **kw):
        import io
        return _RestrictedUnpickler(io.BytesIO(b), **kw).load()


def load_lightning_checkpoint(path, map_location="cpu"):
    return torch.load(path, map_location=map_location, pickle_module=_PickleModule, weights_only=False)


def load_reference_weights(model, path, strict=True, map_location="cpu"):
    """Load `state_dict` of a reference checkpoint into one of our models (same parameter names). Returns the ckpt dict."""
    ckpt = load_lightning_checkpoint(path, map_location=map_location)
    sd = {k: v for k, v in ckpt["state_dict"].items()}
    model.load_state_dict(sd, strict=strict)
    return ckpt


class ModelCheckpoint:
    """Stand-in for the class Lightning keys ModelCheckpoint's state by in `callbacks`; `save_lightning_checkpoint` pickles it
    under the global name `pytorch_lightning.callbacks.model_checkpoint.ModelCheckpoint`.  Never instantiated."""


_PICKLED_AS = {"ModelCheckpoint": "pytorch_lightning.callbacks.model_checkpoint"}


def model_checkpoint_state(ckpt):
    """The ModelCheckpoint entry of a checkpoint's `callbacks` (ours or Lightning's), or None."""
    for key, value in (ckpt.get("callbacks") or {}).items():
        if getattr(key, "__name__", key) == "ModelCheckpoint":
            return value
    return None


def save_lightning_checkpoint(model, path, epoch=0, global_step=0, optimizer_states=None, lr_schedulers=None, extra_state_dict=None,
                              callbacks=None):
    """Write `model` in the layout of the reference's Lightning-1.3.8 checkpoints (SURVEY.md §8b), so that the reference's
    own `Model.load_from_checkpoint(path, config=cfg)` / `--checkpoint` (main.py:67-70,78-79) reads it back:

        state_dict                 parameter / buffer names exactly as the reference's modules name them
        hyper_parameters           {"config": EasyDict(...)} — pickled under the global name `easydict.EasyDict`
        epoch, global_step, pytorch-lightning_version ("1.3.8"), optimizer_states, lr_schedulers, callbacks

    `extra_state_dict`: entries of the reference's parameter-free metric modules (`prec.*`, `success.*`: torchmetrics buffers)
    to carry over from a loaded checkpoint; they hold no weights and are absent by default (Lightning loads non-strictly
    only if asked, so pass them through when the file must load with `strict=True` in the reference).
    `callbacks`: {ModelCheckpoint: state dict} as trainer.Trainer writes it (default: empty)."""
    import sys
    import types
    from .compat import easydict as _ed
    sd = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    if extra_state_dict:
        sd.update({k: v.detach().cpu().clone() for k, v in extra_state_dict.items()})
    cfg = getattr(model, "config", None)
    hp = dict(getattr(model, "hparams", {}) or {})
    if cfg is not None:
        hp["config"] = _ed.EasyDict(dict(cfg))
    ckpt = {"epoch": int(epoch), "global_step": int(global_step), "pytorch-lightning_version": "1.3.8", "state_dict": sd,
            "hyper_parameters": hp, "optimizer_states": optimizer_states or [], "lr_schedulers": lr_schedulers or [],
            "callbacks": callbacks or {}}
    # the stand-ins must be written under the names the reference environment resolves: easydict.EasyDict and Lightning's
    # ModelCheckpoint; pickle checks a global name by importing its module, so each module and its parents are stubbed
    renamed, stubbed = [], {}
    for cls, module in ((_ed.EasyDict, "easydict"), (ModelCheckpoint, _PICKLED_AS["ModelCheckpoint"])):
        if cls.__module__ == module:
            continue
        renamed.append((cls, cls.__module__, cls.__qualname__))
        cls.__module__, cls.__qualname__ = module, cls.__name__
        parts = module.split(".")
        for i in range(1, len(parts) + 1):
            name = ".".join(parts[:i])
            if name not in stubbed:
                stubbed[name] = sys.modules.get(name)
                sys.modules[name] = types.ModuleType(name)
        setattr(sys.modules[module], cls.__name__, cls)
    try:
        torch.save(ckpt, path, _use_new_zipfile_serialization=False)      # the legacy (non-zip) format Lightning 1.3.8 wrote
    finally:
        for cls, module, qualname in renamed:
            cls.__module__, cls.__qualname__ = module, qualname
        for name, old in stubbed.items():
            if old is None:
                sys.modules.pop(name, None)
            else:
                sys.modules[name] = old
    return path
