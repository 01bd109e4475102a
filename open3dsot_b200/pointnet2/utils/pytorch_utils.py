"""Layer builders with the reference's module tree and parameter names.

Mirror of pointnet2/utils/pytorch_utils.py: `SharedMLP` (:12-37), `_BNBase`/`BatchNorm{1,2,3}d` (:40-65),
`_ConvBase`/`Conv{1,2,3}d` (:68-223), `FC` (:226-261), `BNMomentumScheduler` (:272-297), `Seq` (:300-457).
What matters for drop-in use is the *state-dict surface* (SURVEY.md §8b):
    <mlp>.layer{i}.conv.weight, <mlp>.layer{i}.bn.bn.{weight,bias,running_mean,running_var,num_batches_tracked}
    <seq>.{i}.conv.{weight,bias}, <seq>.{i}.bn.bn.*
and the construction rules: bias only when no BN, kaiming-normal conv weights, BN gamma=1 / beta=0.
The classes are plain containers; the native modules read their parameters and run the fused sm_90a
kernels (open3dsot_b200/fused.py) instead of iterating the container.
"""
from typing import List

import torch.nn as nn

_CONV = {1: nn.Conv1d, 2: nn.Conv2d, 3: nn.Conv3d}
_BN = {1: nn.BatchNorm1d, 2: nn.BatchNorm2d, 3: nn.BatchNorm3d}


class _BNBase(nn.Sequential):
    def __init__(self, in_size, batch_norm=None, name=""):
        super().__init__()
        self.add_module(name + "bn", batch_norm(in_size))
        nn.init.constant_(self[0].weight, 1.0)
        nn.init.constant_(self[0].bias, 0)


class BatchNorm1d(_BNBase):
    def __init__(self, in_size: int, *, name: str = ""):
        super().__init__(in_size, batch_norm=nn.BatchNorm1d, name=name)


class BatchNorm2d(_BNBase):
    def __init__(self, in_size: int, name: str = ""):
        super().__init__(in_size, batch_norm=nn.BatchNorm2d, name=name)


class BatchNorm3d(_BNBase):
    def __init__(self, in_size: int, name: str = ""):
        super().__init__(in_size, batch_norm=nn.BatchNorm3d, name=name)


_BN_WRAP = {1: BatchNorm1d, 2: BatchNorm2d, 3: BatchNorm3d}


class _ConvBase(nn.Sequential):
    """conv -> [bn] -> [activation]  (or bn -> activation -> conv when `preact`)."""

    def __init__(self, in_size, out_size, kernel_size, stride, padding, activation, bn, init, conv=None,
                 batch_norm=None, bias=True, preact=False, name=""):
        super().__init__()
        bias = bias and (not bn)
        unit = conv(in_size, out_size, kernel_size=kernel_size, stride=stride, padding=padding, bias=bias)
        init(unit.weight)
        if bias:
            nn.init.constant_(unit.bias, 0)
        pre, post = [], []
        norm_act = []
        if bn:
            norm_act.append((name + "bn", batch_norm(in_size if preact else out_size)))
        if activation is not None:
            norm_act.append((name + "activation", activation))
        (pre if preact else post).extend(norm_act)
        for n, m in pre + [(name + "conv", unit)] + post:
            self.add_module(n, m)


def _conv_class(dim, default_k):
    class _Conv(_ConvBase):
        def __init__(self, in_size: int, out_size: int, *, kernel_size=default_k, stride=None, padding=None,
                     activation=nn.ReLU(inplace=True), bn: bool = False, init=nn.init.kaiming_normal_,
                     bias: bool = True, preact: bool = False, name: str = ""):
            one = 1 if dim == 1 else (1,) * dim
            zero = 0 if dim == 1 else (0,) * dim
            super().__init__(in_size, out_size, kernel_size, one if stride is None else stride,
                             zero if padding is None else padding, activation, bn, init, conv=_CONV[dim],
                             batch_norm=_BN_WRAP[dim], bias=bias, preact=preact, name=name)

    _Conv.__name__ = _Conv.__qualname__ = f"Conv{dim}d"
    return _Conv


Conv1d = _conv_class(1, 1)
Conv2d = _conv_class(2, (1, 1))
Conv3d = _conv_class(3, (1, 1, 1))


class SharedMLP(nn.Sequential):
    """Stack of 1x1 Conv2d(+BN+ReLU) units named `layer{i}`."""

    def __init__(self, args: List[int], *, bn: bool = False, activation=nn.ReLU(inplace=True), preact: bool = False,
                 first: bool = False, name: str = ""):
        super().__init__()
        for i in range(len(args) - 1):
            plain = (not first) or (not preact) or (i != 0)
            self.add_module(name + "layer{}".format(i),
                            Conv2d(args[i], args[i + 1], bn=plain and bn, activation=activation if plain else None,
                                   preact=preact))


class FC(nn.Sequential):
    def __init__(self, in_size: int, out_size: int, *, activation=nn.ReLU(inplace=True), bn: bool = False, init=None,
                 preact: bool = False, name: str = ""):
        super().__init__()
        fc = nn.Linear(in_size, out_size, bias=not bn)
        if init is not None:
            init(fc.weight)
        if not bn:
            nn.init.constant_(fc.bias, 0)
        norm_act = []
        if bn:
            norm_act.append((name + "bn", BatchNorm1d(in_size if preact else out_size)))
        if activation is not None:
            norm_act.append((name + "activation", activation))
        mods = norm_act + [(name + "fc", fc)] if preact else [(name + "fc", fc)] + norm_act
        for n, m in mods:
            self.add_module(n, m)


def set_bn_momentum_default(bn_momentum):
    def fn(m):
        if isinstance(m, (nn.BatchNorm1d, nn.BatchNorm2d, nn.BatchNorm3d)):
            m.momentum = bn_momentum

    return fn


class BNMomentumScheduler(object):
    def __init__(self, model, bn_lambda, last_epoch=-1, setter=set_bn_momentum_default):
        if not isinstance(model, nn.Module):
            raise RuntimeError("Class '{}' is not a PyTorch nn Module".format(type(model).__name__))
        self.model, self.setter, self.lmbd = model, setter, bn_lambda
        self.step(last_epoch + 1)
        self.last_epoch = last_epoch

    def step(self, epoch=None):
        if epoch is None:
            epoch = self.last_epoch + 1
        self.last_epoch = epoch
        self.model.apply(self.setter(self.lmbd(epoch)))


class Seq(nn.Sequential):
    """Fluent builder; children are named "0", "1", ... in call order."""

    def __init__(self, input_channels):
        super().__init__()
        self.count = 0
        self.current_channels = input_channels

    def _push(self, module, out_size=None):
        self.add_module(str(self.count), module)
        self.count += 1
        if out_size is not None:
            self.current_channels = out_size
        return self

    def _conv(self, cls, out_size, kw):
        kw.pop("dilation", None)
        kw.pop("norm_layer", None)
        return self._push(cls(self.current_channels, out_size, **kw), out_size)

    def conv1d(self, out_size: int, **kw):
        return self._conv(Conv1d, out_size, kw)

    def conv2d(self, out_size: int, **kw):
        return self._conv(Conv2d, out_size, kw)

    def conv3d(self, out_size: int, **kw):
        return self._conv(Conv3d, out_size, kw)

    def fc(self, out_size: int, **kw):
        return self._push(FC(self.current_channels, out_size, **kw), out_size)

    def dropout(self, p=0.5):
        return self._push(nn.Dropout(p=0.5))  # the reference ignores `p` (pytorch_utils.py:433)

    def maxpool2d(self, kernel_size, stride=None, padding=0, dilation=1, return_indices=False, ceil_mode=False):
        return self._push(nn.MaxPool2d(kernel_size=kernel_size, stride=stride, padding=padding, dilation=dilation,
                                       return_indices=return_indices, ceil_mode=ceil_mode))
