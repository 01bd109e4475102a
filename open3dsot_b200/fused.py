"""Fused execution of the reference's MLP stacks on the sm_90a point-wise kernels (csrc/pwmlp.cu).

A *stack* is what the reference builds with `pt_utils.SharedMLP` / `pt_utils.Seq` / a bare `nn.Conv1d`:
a chain of 1x1 convolutions, each optionally followed by BatchNorm and ReLU, optionally ending in a max over
groups of S consecutive positions (SA max-pool over nsample — pointnet2_modules.py:70-73; BoxAware max over k —
xcorr.py:100; P2B max over template points — xcorr.py:49).  `mlp_stack` runs such a chain as

    per layer:  o3d_pw_fwd (GEMM + BN statistics [+ pooling] in the epilogue)  ->  o3d_bn_fwd_finalize
    backward :  o3d_pool_bwd_prep | o3d_dense_bwd_prep  ->  per layer  o3d_bn_bwd_finalize, o3d_pw_wgrad, o3d_pw_dgrad

on channels-last activations; normalised activations, the BN backward and the ReLU masks live only inside the
operand loaders / epilogues of the GEMMs.  Parameters stay in the reference's modules (same names, same
state-dict), torch is used for buffers and the autograd graph only.
"""
import ctypes

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _lib, ops, runtime
from .pointnet2.utils import pointnet2_utils

_call = ops._call
_stream = ops._stream


def _r4(n):
    return (n + 3) & ~3


def _ptr(t):
    return None if t is None else t.data_ptr()


# ---------------------------------------------------------------------------------------------- layer parsing
class _LayerSpec:
    __slots__ = ("weight", "bias", "bn", "relu", "lift_c0")

    def __init__(self, weight, bias, bn, relu, lift_c0=0):
        self.weight, self.bias, self.bn, self.relu, self.lift_c0 = weight, bias, bn, relu, lift_c0


def _spec_from_unit(unit):
    """unit: pt_utils._ConvBase (children conv / bn / activation), nn.ConvNd, or nn.Linear."""
    if isinstance(unit, (nn.Conv1d, nn.Conv2d, nn.Conv3d, nn.Linear)):
        return _LayerSpec(unit.weight, unit.bias, None, False)
    conv = getattr(unit, "conv", None)
    if conv is None:
        raise TypeError(f"cannot fuse {type(unit).__name__}")
    bn = getattr(unit, "bn", None)
    if bn is not None and not isinstance(bn, nn.modules.batchnorm._BatchNorm):
        bn = bn[0]  # _BNBase wrapper -> the torch BatchNorm inside
    return _LayerSpec(conv.weight, conv.bias, bn, hasattr(unit, "activation"))


def parse_stack(module):
    """SharedMLP / Seq (children are _ConvBase units), bare conv, or nn.Sequential(conv, BN, ReLU, ...)."""
    if isinstance(module, (nn.Conv1d, nn.Conv2d, nn.Conv3d, nn.Linear)):
        return [_spec_from_unit(module)]
    kids = list(module.children())
    if kids and all(hasattr(k, "conv") for k in kids):
        return [_spec_from_unit(k) for k in kids]
    specs = []
    for k in kids:  # flat torch Sequential: conv / linear, then optional BatchNorm, then optional ReLU
        if isinstance(k, (nn.Conv1d, nn.Conv2d, nn.Linear)):
            specs.append(_LayerSpec(k.weight, k.bias, None, False))
        elif isinstance(k, nn.modules.batchnorm._BatchNorm):
            specs[-1].bn = k
        elif isinstance(k, nn.ReLU):
            specs[-1].relu = True
        else:
            raise TypeError(f"cannot fuse {type(k).__name__} inside {type(module).__name__}")
    return specs


# ---------------------------------------------------------------------------------------------- the autograd op
def _tracks_stats(bn):
    return bn is not None and bn.track_running_stats and bn.running_mean is not None


class _Meta:
    """Static description of one stack invocation (python objects only), with the stack's flat parameter list
    ([weight, bias, gamma, beta] per layer, None where a layer has no such tensor) and the running BatchNorm statistics."""

    def __init__(self, specs, S, training, xyz_first=False, c0=0, dx_cols=0):
        if len(specs) > _lib.MAX_LAYERS:
            raise RuntimeError(f"fused MLP stack: at most {_lib.MAX_LAYERS} layers")
        self.n = len(specs)
        self.S = int(S)
        self.training = bool(training)
        self.xyz_first = bool(xyz_first)
        self.c0 = int(c0)
        self.dx_cols = int(dx_cols)
        self.grad_mode = torch.is_grad_enabled()   # of the CALLER (inside Function.forward grad mode is always off)
        self.bns = [s.bn for s in specs]
        self.relu = [bool(s.relu) for s in specs]
        # a spec without weight is the lifted first layer (BatchNorm / ReLU only; `lift_c0` output channels)
        self.cout = [s.weight.shape[0] if s.weight is not None else s.lift_c0 for s in specs]
        self.cin = [s.weight.numel() // s.weight.shape[0] if s.weight is not None else 0 for s in specs]
        self.params = []
        for s in specs:
            self.params += [s.weight, s.bias, s.bn.weight if s.bn is not None else None, s.bn.bias if s.bn is not None else None]
        self.stats = [t for bn in self.bns if _tracks_stats(bn) for t in (bn.running_mean, bn.running_var)]


def _describe(meta, P, K0, params):
    """the StackDesc of `meta` over `params` (meta.params, or the same tensors as received by the autograd function)"""
    d = _lib.StackDesc()
    d.n_layers, d.P, d.K0, d.S = meta.n, P, K0, meta.S
    d.training, d.use_tc = int(meta.training), int(runtime.tc_level())
    d.xyz_first, d.c0, d.dx_cols = int(meta.xyz_first), meta.c0, meta.dx_cols
    for l in range(meta.n):
        W, b, g, be = params[4 * l:4 * l + 4]
        bn = meta.bns[l]
        d.cin[l], d.cout[l], d.relu[l], d.has_bn[l] = meta.cin[l], meta.cout[l], int(meta.relu[l]), int(bn is not None)
        d.weight[l], d.bias[l], d.gamma[l], d.beta[l] = _ptr(W), _ptr(b), _ptr(g), _ptr(be)
        if bn is not None:
            d.momentum[l] = 0.1 if bn.momentum is None else bn.momentum
            d.eps[l] = bn.eps
            if _tracks_stats(bn):
                d.running_mean[l], d.running_var[l] = bn.running_mean.data_ptr(), bn.running_var.data_ptr()
                d.num_batches_tracked[l] = bn.num_batches_tracked.data_ptr()
    return d


def _static_cached(tag, extra, deps, make):
    """`make()` -- a tensor computed from the tensors `deps` (None entries allowed) -- cached for inference with static weights
    (runtime.static_weights_scope).  The entry is stored on the first tensor of `deps`, keyed by `tag`, `extra` and the identity
    of every dep, and is valid while every dep's version and the weights generation (advanced by every training step, whose
    writes bump no version) are unchanged (`load_state_dict` / in-place edits / training invalidate it).  It keeps its deps
    alive, so their ids stay unique.

    A cached tensor may be read from another stream (the template / search branches run side by side, run_ahead) with no
    ordering against the stream that built it, so the builder finishes before the entry becomes visible.  During graph capture
    nothing is cached: a missing value is built privately, as part of the graph.  Either way the caller keeps the returned
    tensor referenced until the kernel that reads it is enqueued."""
    owner = next(t for t in deps if t is not None)
    cache = owner.__dict__.setdefault("_o3d_static", {})
    key = (tag, extra, tuple(id(t) for t in deps))
    versions = (runtime.weights_generation(),) + tuple(-1 if t is None else t._version for t in deps)
    hit = cache.get(key)
    if hit is not None and hit[0] == versions:
        return hit[1]
    value = make()
    if not torch.cuda.is_current_stream_capturing():
        torch.cuda.current_stream().synchronize()
        cache[key] = (versions, value, deps)
    return value


def _derived(weight, tag, make):
    """A tensor computed from `weight` (e.g. a contiguous column slice).  With static weights and no autograd it is built once
    and cached on the weight, which also keeps its address stable for the prepared-block cache."""
    if not runtime.static_weights() or torch.is_grad_enabled():
        return make()
    return _static_cached(tag, None, [weight], lambda: make().detach())


def _precision_code(training, need_grad):
    """o3d_stack_t.precision of a forward under the current runtime.inference_precision() and, for a stack in training mode,
    runtime.training_precision(); bf16 inference refuses autograd and training"""
    if runtime.inference_precision() == "fp32":
        if training and runtime.training_precision() == "bf16":
            return _lib.PRECISION_BF16_TRAIN
        return _lib.PRECISION_TF32X3
    if need_grad or training:
        raise RuntimeError("bf16 inference precision: forward passes that need a gradient, and modules in training mode, run in "
                           "fp32 only (leave runtime.inference_precision_scope('bf16'))")
    return _lib.PRECISION_BF16


def _prepare_stack(d, device):
    """the stack's prepared block: packed weights and folded running statistics (o3d_stack_prepare)"""
    L = _lib.lib()
    nbytes = L.o3d_stack_prepared_bytes(ctypes.byref(d))
    if nbytes < 0:
        raise RuntimeError("fused MLP stack: invalid stack description")
    block = torch.empty(max(int(nbytes), 16), dtype=torch.uint8, device=device)
    _lib.check(L.o3d_stack_prepare(ctypes.byref(d), block.data_ptr(), _stream()), "o3d_stack_prepare")
    return block


def _param_grad_targets(needs, d, meta):
    """Where a stack's backward writes its parameter gradients (`needs`: needs_input_grad of meta.params).  Default: fresh
    tensors returned to autograd.  Inside `runtime.grad_inplace_scope()` and when EVERY parameter that needs a gradient is a leaf
    with a pre-allocated contiguous `.grad` (the engine's flat bucket): the kernels add into those buffers directly and autograd
    gets None for them."""
    params = meta.params
    need = [i for i, t in enumerate(params) if t is not None and needs[i]]
    inplace = runtime.grad_inplace() and bool(need) and all(
        params[i].is_leaf and params[i].grad is not None and params[i].grad.is_contiguous() and params[i].grad.dtype == torch.float32
        for i in need)
    grads = [None] * len(params)
    fields = (d.d_weight, d.d_bias, d.d_gamma, d.d_beta)           # params[i] is field i % 4 of layer i // 4
    for i in range(len(params)):
        fields[i % 4][i // 4] = None
    for i in need:
        if not inplace:
            grads[i] = torch.empty_like(params[i])
        fields[i % 4][i // 4] = (params[i].grad if inplace else grads[i]).data_ptr()
    d.accumulate = int(inplace)
    return grads


class _LiftGeom:
    """Static geometry of a lifted stack: Y0[p] = Z[cloud(p) * rows_per_cloud + (ridx[p] | p % ridx_mod)] + s[p] . u, with c0
    channels."""
    __slots__ = ("P", "ridx_mod", "rows_per_cloud", "pos_per_cloud", "grp", "c0")

    def __init__(self, P, ridx_mod, rows_per_cloud, pos_per_cloud, grp, c0):
        self.P, self.ridx_mod, self.rows_per_cloud, self.pos_per_cloud, self.grp = P, ridx_mod, rows_per_cloud, pos_per_cloud, grp
        self.c0 = c0


class _StackFn(torch.autograd.Function):
    """One stack; params = meta.params.  Plain (lift None): x (P, K0) channels-last fp32.  Lifted (lift a _LiftGeom, x None): the
    first 1x1 convolution has been split (include/o3d_b200.h `o3d_lift_t`) into its feature part applied to the SOURCE points
    (z = W0_f . rows, an ordinary one-layer stack) and gathered, plus up to four per-position scalars s with weight rows u:
    z (rows, c0) | None, ridx (P,) int32 | None, s (P, 4) | None, u (4, c0) | None; layer 0 = (None, None, gamma0, beta0)."""

    @staticmethod
    def forward(ctx, meta, lift, x, z, ridx, s, u, *params):
        for t in (x, z, ridx, s, u) + params:
            if t is not None and not t.is_contiguous():
                raise RuntimeError("fused MLP stack: tensors must be contiguous")
        P, K0 = x.shape if lift is None else (lift.P, lift.c0)
        dev = next(t for t in (x, z, s) if t is not None).device
        d = _describe(meta, P, K0, params)
        lf = None
        if lift is not None:
            lf = _lib.LiftDesc()
            lf.z, lf.ldz, lf.ridx, lf.ridx_mod = _ptr(z), lift.c0, _ptr(ridx), lift.ridx_mod
            lf.rows_per_cloud, lf.pos_per_cloud, lf.grp = lift.rows_per_cloud, lift.pos_per_cloud, lift.grp
            lf.s, lf.u = _ptr(s), _ptr(u)
            d.lift = ctypes.pointer(lf)
        L = _lib.lib()
        if runtime.recording_stack_rows():
            th = (ctypes.c_int * 4)()
            n = L.o3d_stack_plan_thresholds(ctypes.byref(d), th)
            if n < 0:
                raise RuntimeError("fused MLP stack: invalid stack description")
            runtime.note_stack_rows(P, th[:n])
        need_grad = meta.grad_mode and any(ctx.needs_input_grad)   # (needs_input_grad mirrors requires_grad even under no_grad)
        d.precision = _precision_code(meta.training, need_grad)
        block = None            # inference with static weights: the prepared block, referenced here until the forward is enqueued
        if not need_grad and not meta.training and runtime.static_weights():
            lifted = False if lift is None else (z is not None, s is not None)
            shape = (P, K0, meta.S, lifted, runtime.tc_level(), meta.xyz_first, meta.c0, d.precision)
            block = _static_cached("stack", shape, meta.params + meta.stats, lambda: _prepare_stack(d, dev))
            d.prepared = block.data_ptr()
        nbytes = L.o3d_stack_workspace_bytes(ctypes.byref(d), 0)
        if nbytes < 0:
            raise RuntimeError("fused MLP stack: invalid stack description")
        ws = torch.empty(max(int(nbytes), 16), dtype=torch.uint8, device=dev)
        rows = P // meta.S if meta.S > 0 else P
        Nw, Cout = _r4(meta.cout[-1]), meta.cout[-1]
        out = torch.empty(rows, Nw, dtype=torch.float32, device=dev)
        ops.LAUNCHES += 3 * meta.n + 1
        _lib.check(L.o3d_stack_forward(ctypes.byref(d), _ptr(x), ws.data_ptr(), out.data_ptr(), int(need_grad), _stream()),
                   "o3d_stack_forward")
        if need_grad:
            ctx.meta, ctx.desc, ctx.lf = meta, d, lf     # the backward writes d_z / d_s / d_u into lf
            ctx.save_for_backward(x, z, ridx, s, u, ws, out)
        return out if Nw == Cout else out[:, :Cout]

    @staticmethod
    def backward(ctx, dout):
        meta, d, lf = ctx.meta, ctx.desc, ctx.lf
        x, z, ridx, s, u, ws, out = ctx.saved_tensors
        if dout.shape[1] != out.shape[1] or not dout.is_contiguous():
            dpad = torch.zeros(out.shape, dtype=torch.float32, device=out.device)
            dpad[:, :dout.shape[1]] = dout
            dout = dpad
        need = ctx.needs_input_grad                     # False for inputs that are None
        grads = _param_grad_targets(need[7:], d, meta)
        dx = torch.empty_like(x) if need[2] else None
        dz, ds, du = (torch.zeros_like(t) if need[i] else None for i, t in ((3, z), (5, s), (6, u)))
        if lf is not None:
            lf.d_z, lf.d_s, lf.d_u = _ptr(dz), _ptr(ds), _ptr(du)
        L = _lib.lib()
        nbytes = L.o3d_stack_workspace_bytes(ctypes.byref(d), 1)
        wb = torch.empty(max(int(nbytes), 16), dtype=torch.uint8, device=out.device)
        ops.LAUNCHES += 5 * meta.n + 1
        _lib.check(L.o3d_stack_backward(ctypes.byref(d), _ptr(x), ws.data_ptr(), wb.data_ptr(), out.data_ptr(), dout.data_ptr(),
                                        _ptr(dx), _stream()), "o3d_stack_backward")
        return (None, None, dx, dz, None, ds, du, *grads)


def lifted_stack(specs, geom, z=None, ridx=None, s=None, u=None, S=0, training=True):
    """specs[0] is the lifted layer: its conv has ALREADY been applied (z, s.u); only its BatchNorm / ReLU remain."""
    meta = _Meta([_LayerSpec(None, None, specs[0].bn, specs[0].relu, lift_c0=geom.c0)] + list(specs[1:]), S, training)
    return _StackFn.apply(meta, geom, None, z, ridx, s, u, *meta.params)


def _pow2_divisor(n, cap=64):
    g = 1
    while g * 2 <= cap and n % (g * 2) == 0:
        g *= 2
    return g


def _liftable(specs):
    """The first conv can be lifted when another layer follows it, its output width is a multiple of 4, and lifting is on."""
    return runtime.lift_enabled() and len(specs) >= 2 and specs[0].weight.shape[0] % 4 == 0


def mlp_stack(x2d, specs, S=0, training=True, xyz_first=False, c0=0, dx_cols=0):
    """Run a stack on a channels-last matrix.

    x2d        (P, K0) fp32, contiguous, K0 % 4 == 0 (zero-padded input channels)
    specs      list of _LayerSpec (parameters of the reference modules, checkpoint layout)
    S          pooling group size over consecutive positions (0 = dense output); must divide 128 and P
    xyz_first  layer-0 weight columns are [xyz(3) | features(c0)] while rows are [features | dx dy dz 0]
    dx_cols    backward only needs the gradient of the first dx_cols input columns (0 = all)
    returns    (P or P//S, Cout_last)
    """
    if not x2d.is_cuda:
        raise RuntimeError("open3dsot_b200.fused: CUDA tensors required (there is no CPU path)")
    assert x2d.dim() == 2 and x2d.is_contiguous() and x2d.dtype == torch.float32 and x2d.shape[1] % 4 == 0
    meta = _Meta(specs, S, training, xyz_first, c0, dx_cols)
    return _StackFn.apply(meta, None, x2d, None, None, None, None, *meta.params)


# ---------------------------------------------------------------------------------------------- layout helpers
def to_channels_last(feat, pad_to4=True):
    """(B, C, N) [any strides] -> (B, N, Cp) contiguous with Cp = round_up(C, 4) (zero padded)."""
    cl = feat.transpose(1, 2)
    C = cl.shape[2]
    Cp = _r4(C) if pad_to4 else C
    if Cp != C:
        cl = F.pad(cl, (0, Cp - C))
    return cl.contiguous()


def from_channels_last(cl):
    """(B, N, C) contiguous -> (B, C, N) view (no copy); consumers that want channels-last undo it for free."""
    return cl.transpose(1, 2)


# ---------------------------------------------------------------------------------------------- single-kernel SA layer (inference)
def _sa_fused_ok(specs, S, npoint, N, C):
    """shape range of o3d_sa_fused_forward (csrc/sa_fused.cu): nsample | 64, <= 256 channels per layer, BatchNorm with running stats"""
    if not runtime.sa_fused_enabled() or runtime.CHOICE_HOOK is not None or not runtime.fused_enabled():
        return False
    if S < 1 or 64 % S != 0 or npoint % (64 // S) != 0 or C > 288 or N * 12 > 96 * 1024 or len(specs) > _lib.MAX_LAYERS:
        return False
    for s in specs:
        if s.weight is None or s.weight.shape[0] > 256:
            return False
        if s.bn is not None and not _tracks_stats(s.bn):
            return False
    return specs[0].weight.numel() // specs[0].weight.shape[0] == C + 3


def _sa_fused_prepare(d, device):
    """the layer's parameter block: pre-tiled weight images, folded BatchNorm"""
    L = _lib.lib()
    nbytes = L.o3d_sa_fused_prepared_bytes(ctypes.byref(d))
    if nbytes < 0:
        raise RuntimeError("fused SA layer: SharedMLP outside the kernel's range")
    block = torch.empty(int(nbytes), dtype=torch.uint8, device=device)
    _lib.check(L.o3d_sa_fused_prepare(ctypes.byref(d), block.data_ptr(), _stream()), "o3d_sa_fused_prepare")
    return block


def _sa_fused_forward(specs, xyz, new_xyz, feat_cl, C, radius, S, normalize):
    """one kernel: ball query + grouping + SharedMLP (running-statistics BatchNorm, ReLU) + max-pool -> (B, npoint, Cout) channels-last"""
    B, N, _ = xyz.shape
    npoint = new_xyz.shape[1]
    meta = _Meta(specs, S, False, xyz_first=True, c0=C)
    d = _describe(meta, B * npoint * S, _r4(C) + 4, meta.params)
    d.precision = _precision_code(False, False)
    if runtime.static_weights():
        block = _static_cached("sa_fused", d.precision, meta.params + meta.stats, lambda: _sa_fused_prepare(d, xyz.device))
    else:
        block = _sa_fused_prepare(d, xyz.device)
    ldo = _r4(meta.cout[-1])
    out = torch.empty(B, npoint, ldo, dtype=torch.float32, device=xyz.device)
    _lib.check(_lib.lib().o3d_sa_fused_forward(ctypes.byref(d), block.data_ptr(), xyz.data_ptr(), new_xyz.data_ptr(), _ptr(feat_cl),
                                               0 if feat_cl is None else feat_cl.shape[2], B, N, npoint, float(radius), S,
                                               int(bool(normalize)), out.data_ptr(), ldo, None, _stream()), "o3d_sa_fused_forward")
    return out if ldo == meta.cout[-1] else out[:, :, :meta.cout[-1]]


# ---------------------------------------------------------------------------------------------- modules
def seq_forward(module, x):
    """Seq / SharedMLP-on-1D / bare Conv1d applied to x (B, C, L) -> (B, Cout, L) (channels-last view)."""
    B, C, L = x.shape
    cl = to_channels_last(x)
    specs = parse_stack(module)
    out = mlp_stack(cl.view(B * L, cl.shape[2]), specs, 0, module.training)
    return from_channels_last(out.reshape(B, L, out.shape[1]))


def sa_forward(sa, xyz, features, sample_idxs):
    """Fused body of _PointnetSAModuleBase.forward (pointnet2_modules.py:58-76) for every (grouper, mlp) scale."""
    B, N, _ = xyz.shape
    npoint = sample_idxs.shape[1]
    if sa.use_fps:
        new_xyz = torch.gather(xyz, 1, sample_idxs.long().unsqueeze(-1).expand(-1, -1, 3)).contiguous()
    else:
        new_xyz = xyz[:, :npoint].contiguous()
    feat_cl, C = None, 0
    if features is not None:
        C = features.shape[1]
        feat_cl = to_channels_last(features)
    Cp = 0 if feat_cl is None else feat_cl.shape[2]
    outs = []
    for grouper, mlp in zip(sa.groupers, sa.mlps):
        S = grouper.nsample
        if 128 % S != 0:
            raise RuntimeError(f"fused SA layer: nsample={S} must divide 128")
        specs = parse_stack(mlp)
        if not grouper.use_xyz:
            raise RuntimeError("fused SA layer expects use_xyz=True (every shipped model does)")
        need_xyz = torch.is_grad_enabled() and (xyz.requires_grad or new_xyz.requires_grad)
        if not sa.training and not torch.is_grad_enabled() and _sa_fused_ok(specs, S, npoint, N, C):
            xyz_c = xyz if xyz.is_contiguous() else xyz.contiguous()
            pooled = _sa_fused_forward(specs, xyz_c, new_xyz, feat_cl, C, grouper.radius, S, grouper.normalize_xyz)
            outs.append(from_channels_last(pooled))
            continue
        if _liftable(specs) and (specs[0].bias is None or feat_cl is not None):
            # Lifted first layer: W0 . [x(idx) - c, f(idx)] = (W0_f . f)[idx] + W0_x . (x(idx) - c) — the feature part of the
            # convolution runs once per SOURCE point (z) and is gathered; the relative coordinates (dx, dy, dz) are applied per
            # position, directly (same difference-then-multiply arithmetic as the reference).  The grouped
            # (B, 3+C, npoint, nsample) tensor never exists (pointnet2_utils.py:317-329 + the first SharedMLP layer,
            # pointnet2_modules.py:64-69).
            W0 = specs[0].weight
            C0 = W0.shape[0]
            W2 = W0.reshape(C0, -1)
            if runtime.CHOICE_HOOK is None:
                # fused ball query + relative coordinates: grouped (B, npoint, S, 4) = [dx dy dz 0], idx (B, npoint, S)
                rel, idx = pointnet2_utils.query_and_group_cl(xyz, new_xyz, None, grouper.radius, S, grouper.normalize_xyz)
            else:   # parity tests: record / substitute the discrete choice, relative coordinates by plain indexing
                idx = runtime.choose("ball_query", {"radius": grouper.radius, "nsample": S, "N": N, "npoint": npoint},
                                     lambda: pointnet2_utils.ball_query(grouper.radius, S, xyz, new_xyz))
                rel = xyz.gather(1, idx.long().view(B, -1, 1).expand(-1, -1, 3)).view(B, npoint, S, 3) - new_xyz.unsqueeze(2)
                if grouper.normalize_xyz:
                    rel = rel / grouper.radius
                rel = F.pad(rel, (0, 1)).contiguous()
            u = _derived(W0, "u_xyz", lambda: F.pad(W2[:, :3].t(), (0, 0, 0, 1)).contiguous())   # (4, C0): rows = W0's xyz columns, 0
            z = None
            if feat_cl is not None:
                Wf = _derived(W0, "w_feat", lambda: W2[:, 3:].contiguous())
                z = mlp_stack(feat_cl.view(B * N, Cp), [_LayerSpec(Wf, specs[0].bias, None, False)], 0, sa.training)
            geom = _LiftGeom(B * npoint * S, 0, N, npoint * S, S, C0)
            pooled = lifted_stack(specs, geom, z=z, ridx=idx.view(-1) if z is not None else None,
                                  s=rel.view(B * npoint * S, 4), u=u, S=S, training=sa.training)
        else:
            grouped, _idx = pointnet2_utils.query_and_group_cl(xyz, new_xyz, feat_cl, grouper.radius, S,
                                                               grouper.normalize_xyz)
            # the reference's channel order is [xyz(3), features(C)]; kernel rows are [features(Cp) | dx dy dz 0]:
            # the re-ordering of the first conv's columns happens inside o3d_stack_forward (xyz_first)
            # coordinates that carry no gradient (every backbone layer; not the RPN's votes) spare the backward its
            # (dx,dy,dz) columns
            pooled = mlp_stack(grouped.view(B * npoint * S, Cp + 4), specs, S, sa.training, xyz_first=True, c0=C,
                               dx_cols=0 if (need_xyz or Cp == 0) else Cp)
        outs.append(from_channels_last(pooled.reshape(B, npoint, pooled.shape[1])))
    return new_xyz, outs


class _ThreeNNInterpCL(torch.autograd.Function):
    @staticmethod
    def forward(ctx, unknown, known, known_feat_cl):
        out, idx, w = ops.three_nn_interpolate(unknown, known, known_feat_cl)
        ctx.save_for_backward(idx, w)
        ctx.m = known.shape[1]
        return out

    @staticmethod
    def backward(ctx, g):
        idx, w = ctx.saved_tensors
        return None, None, ops.three_nn_interpolate_grad(g.contiguous(), idx, w, ctx.m)


def fp_forward(fp, unknown, known, unknow_feats, known_feats):
    """Fused PointnetFPModule.forward (pointnet2_modules.py:187-212)."""
    B, n, _ = unknown.shape
    kf = to_channels_last(known_feats)
    C2 = known_feats.shape[1]
    interp = _ThreeNNInterpCL.apply(unknown.contiguous(), known.contiguous(), kf)[:, :, :C2]
    if unknow_feats is not None:
        cl = torch.cat([interp, unknow_feats.transpose(1, 2)], dim=2)
    else:
        cl = interp
    C = cl.shape[2]
    if C % 4:
        cl = F.pad(cl, (0, _r4(C) - C))
    cl = cl.contiguous()
    out = mlp_stack(cl.view(B * n, cl.shape[2]), parse_stack(fp.mlp), 0, fp.training)
    return from_channels_last(out.reshape(B, n, out.shape[1]))


class _GroupRowsCL(torch.autograd.Function):
    @staticmethod
    def forward(ctx, feat_cl, idx):
        B, N, C = feat_cl.shape
        L = idx.shape[1]
        out = torch.empty(B, L, C, dtype=torch.float32, device=feat_cl.device)
        _call("o3d_group_rows", feat_cl.data_ptr(), idx.data_ptr(), B, N, L, C, out.data_ptr(), _stream())
        ctx.save_for_backward(idx)
        ctx.N = N
        return out

    @staticmethod
    def backward(ctx, g):
        (idx,) = ctx.saved_tensors
        g = g.contiguous()
        B, L, C = g.shape
        gf = torch.zeros(B, ctx.N, C, dtype=torch.float32, device=g.device)
        _call("o3d_group_rows_grad", g.data_ptr(), idx.data_ptr(), B, ctx.N, L, C, gf.data_ptr(), _stream())
        return gf, None


class _P2BCosine(torch.autograd.Function):
    """nn.CosineSimilarity(dim=1) between every (template, search) feature pair (xcorr.py:37-38) -> (B, n2, n1)."""

    @staticmethod
    def forward(ctx, t_cl, s_cl):
        sim, tn, sn = ops.p2b_cosine(t_cl, s_cl)
        ctx.save_for_backward(t_cl, s_cl, sim, tn, sn)
        return sim

    @staticmethod
    def backward(ctx, dsim):
        t_cl, s_cl, sim, tn, sn = ctx.saved_tensors
        dt, ds = ops.p2b_cosine_grad(dsim.contiguous(), sim, t_cl, s_cl, tn, sn, need_t=ctx.needs_input_grad[0],
                                     need_s=ctx.needs_input_grad[1])
        return dt, ds


def boxaware_xcorr_forward(xc, template_feature, search_feature, template_xyz, template_bc, search_bc):
    """Fused BoxAwareXCorr.forward (models/head/xcorr.py:81-103): box-cloud top-k, row gather, MLP + max over k."""
    B, f, M = template_feature.shape
    N = search_bc.shape[1]
    k = xc.k
    if 128 % k != 0:
        raise RuntimeError(f"fused BoxAwareXCorr: k={k} must divide 128")
    # (B,N,k) nearest template box clouds per search point: o3d_xcorr_boxaware_fwd (the reference: cdist + argsort[:k])
    topk = runtime.choose("boxaware_topk", {"k": k, "M": M, "N": N},
                          lambda: ops.boxaware_topk(template_bc.detach().contiguous(), search_bc.detach().contiguous(), k))
    # channel order [xyz(3), bc(9), feat(f)] == the reference's cat order (xcorr.py:82-84)
    tmpl = torch.cat([template_xyz, template_bc, template_feature.transpose(1, 2)], dim=2)
    C = tmpl.shape[2]
    if C % 4:
        tmpl = F.pad(tmpl, (0, _r4(C) - C))
    specs = parse_stack(xc.mlp)
    if _liftable(specs) and (N * k) % 4 == 0:
        # lifted: the first conv runs on the M template rows; the (B, 268, N, k) grouped tensor is never built (xcorr.py:89-98)
        tm = tmpl.contiguous()
        z = mlp_stack(tm.view(B * M, tm.shape[2]), [_LayerSpec(specs[0].weight, specs[0].bias, None, False)], 0, xc.training)
        geom = _LiftGeom(B * N * k, 0, M, N * k, _pow2_divisor(N * k), z.shape[1])
        pooled = lifted_stack(specs, geom, z=z, ridx=topk.view(-1), S=k, training=xc.training)
    else:
        rows = _GroupRowsCL.apply(tmpl.contiguous(), topk.view(B, N * k))                 # (B, N*k, Cp)
        pooled = mlp_stack(rows.view(B * N * k, rows.shape[2]), specs, k, xc.training)
    fusion = from_channels_last(pooled.reshape(B, N, pooled.shape[1]))
    return seq_forward(xc.fea_layer, fusion)


def p2b_xcorr_forward(xc, template_feature, search_feature, template_xyz):
    """Fused P2B_XCorr.forward (models/head/xcorr.py:33-53); positions ordered (b, search j, template i) so that the
    max over the template dimension is a max over groups of n1 consecutive positions."""
    B, f, n1 = template_feature.shape
    n2 = search_feature.shape[2]
    if 128 % n1 != 0:
        raise RuntimeError(f"fused P2B_XCorr: number of template points {n1} must divide 128")
    t_cl = template_feature.transpose(1, 2)                                                        # (B,n1,f)
    sim_t = _P2BCosine.apply(t_cl.contiguous(), search_feature.transpose(1, 2).contiguous())       # (B,n2,n1), eps 1e-8
    sim = sim_t.transpose(1, 2)                                                                    # (B,n1,n2) as the reference
    specs = parse_stack(xc.mlp)
    if _liftable(specs) and (n1 & (n1 - 1)) == 0:
        # lifted: the first conv's input [sim(1), xyz(3), feature(f)] (xcorr.py:39-46) is a per-template row plus ONE scalar
        # per (search, template) pair, so Y0[(b,j,i)] = (W[:,1:] . [xyz_i, f_i]) + sim[b,i,j] * W[:,0] and the
        # (B, 260, n1, n2) fusion tensor is never built
        W0 = specs[0].weight.reshape(specs[0].weight.shape[0], -1)
        rows = torch.cat([template_xyz, t_cl], dim=2)                                               # (B, n1, 3 + f)
        C = rows.shape[2]
        if C % 4:
            rows = F.pad(rows, (0, _r4(C) - C))
        Wr = _derived(specs[0].weight, "w_rest", lambda: W0[:, 1:].contiguous())
        z = mlp_stack(rows.reshape(B * n1, rows.shape[2]), [_LayerSpec(Wr, specs[0].bias, None, False)], 0, xc.training)
        geom = _LiftGeom(B * n2 * n1, n1, n1, n2 * n1, n1, z.shape[1])
        pooled = lifted_stack(specs, geom, z=z, s=F.pad(sim_t.reshape(-1, 1), (0, 3)),
                              u=_derived(specs[0].weight, "u_sim", lambda: F.pad(W0[:, :1].t(), (0, 0, 0, 3)).contiguous()), S=n1,
                              training=xc.training)
    else:
        fusion = torch.cat([sim.transpose(1, 2).unsqueeze(-1),                                      # (B,n2,n1,1)
                            template_xyz.unsqueeze(1).expand(B, n2, n1, 3),
                            t_cl.unsqueeze(1).expand(B, n2, n1, f)], dim=3)
        C = fusion.shape[3]
        if C % 4:
            fusion = F.pad(fusion, (0, _r4(C) - C))
        pooled = mlp_stack(fusion.reshape(B * n2 * n1, fusion.shape[3]), specs, n1, xc.training)
    out = from_channels_last(pooled.reshape(B, n2, pooled.shape[1]))
    return seq_forward(xc.fea_layer, out)


# ---------------------------------------------------------------------------------------------- M2-Track dense nets
def rows_forward(module, x):
    """Linear/BN/ReLU head (nn.Sequential) applied to x (B, C) -> (B, Cout)."""
    C = x.shape[1]
    if C % 4:
        x = F.pad(x, (0, _r4(C) - C))
    return mlp_stack(x.contiguous(), parse_stack(module), 0, module.training)


def _block_specs(blocks):
    """nn.Sequential(Conv1d, BatchNorm1d, ReLU) blocks (models/backbone/pointnet.py:160-181) -> layer specs."""
    return [_LayerSpec(b[0].weight, b[0].bias, b[1], True) for b in blocks]


def _pool_groups(P_per_cloud):
    for s in (64, 32, 16, 8, 4, 2, 1):
        if P_per_cloud % s == 0:
            return s
    return 1


def minipointnet_forward(net, x):
    """Fused MiniPointNet.forward (models/backbone/pointnet.py:91-141): per-point conv/BN/ReLU stack, global max over
    the N points (max over groups of <= 64 positions in the GEMM epilogue, then over the groups), FC/BN/ReLU head."""
    B, C, N = x.shape
    mods = list(net.features)
    cut = next(i for i, m in enumerate(mods) if isinstance(m, nn.AdaptiveMaxPool1d))
    per_point = nn.Sequential(*mods[:cut])
    head = nn.Sequential(*[m for m in mods[cut + 1:] if not isinstance(m, nn.Flatten)])
    per_point.train(net.training)
    head.train(net.training)
    cl = to_channels_last(x)
    S = _pool_groups(N)
    pooled = mlp_stack(cl.view(B * N, cl.shape[2]), parse_stack(per_point), S, net.training)       # (B*N/S, C')
    feat = pooled.view(B, N // S, pooled.shape[1]).max(dim=1)[0]
    if len(list(head.children())):
        feat = mlp_stack(feat.contiguous(), parse_stack(head), 0, net.training)
    if net.output_size > 0:
        feat = mlp_stack(feat.contiguous(), [_LayerSpec(net.fc.weight, net.fc.bias, None, False)], 0, net.training)
    return feat


def segpointnet_forward(net, x):
    """Fused SegPointNet.forward (models/backbone/pointnet.py:183-204)."""
    B, C, N = x.shape
    cl = to_channels_last(x)
    P = B * N
    blocks = list(net.seq_per_point)
    second = mlp_stack(cl.view(P, cl.shape[2]), _block_specs(blocks[:2]), 0, net.training)           # (P, 64)
    S = _pool_groups(N)
    pooled = mlp_stack(second.contiguous(), _block_specs(blocks[2:]), S, net.training)               # (P/S, 1024)
    pooled = pooled.view(B, N // S, pooled.shape[1]).max(dim=1)[0]                                   # (B, 1024)
    cat = torch.cat([second.view(B, N, -1), pooled.unsqueeze(1).expand(B, N, pooled.shape[1])], dim=2)
    Cc = cat.shape[2]
    if Cc % 4:
        cat = F.pad(cat, (0, _r4(Cc) - Cc))
    specs = _block_specs(list(net.seq_per_point2))
    if net.output_size > 0:
        specs.append(_LayerSpec(net.fc.weight, net.fc.bias, None, False))
    out = mlp_stack(cat.reshape(P, cat.shape[2]), specs, 0, net.training)
    out = from_channels_last(out.reshape(B, N, out.shape[1]))
    if net.return_intermediate:
        return out, pooled
    return out


# ---------------------------------------------------------------------------------------------- FPS overlap
_SIDE_STREAMS = {}


def _side_stream(device):
    side = _SIDE_STREAMS.get(device.index)
    if side is None:
        side = _SIDE_STREAMS[device.index] = torch.cuda.Stream(device=device)
    return side


def fps_ahead(points, npoint):
    """Launch furthest-point sampling of `points` (B,N,3+) on a side stream and return (idx, join).  FPS is a serial chain
    of npoint steps that occupies one CTA per cloud (48 of 132 SMs at config 2); started before the template branch it
    runs underneath that branch's GEMMs.  `join()` makes the current stream wait for it (graph-capture safe fork/join)."""
    cur = torch.cuda.current_stream()
    side = _side_stream(points.device)
    xyz = points[..., 0:3].contiguous()
    side.wait_stream(cur)
    with torch.cuda.stream(side):
        idx = pointnet2_utils.furthest_point_sample(xyz, npoint)
    xyz.record_stream(side)
    idx.record_stream(cur)

    def join():
        cur.wait_stream(side)
        return idx
    return join


def _tensors(obj):
    if torch.is_tensor(obj):
        yield obj
    elif isinstance(obj, (tuple, list)):
        for o in obj:
            yield from _tensors(o)


def run_ahead(fn):
    """Inference only (no autograd): run `fn()` — a whole branch of the network, e.g. the template backbone — on the side stream
    and return `join()`, which makes the current stream wait for it and hands over fn's result.  At B = 1 a branch occupies a
    handful of SMs (one CTA per cloud in FPS, 2-8 CTAs per layer), so the template and search branches — independent until the
    cross-correlation — run side by side; inside a captured CUDA graph the fork / join becomes two parallel branches."""
    assert not torch.is_grad_enabled(), "run_ahead is for inference (autograd does not see the stream switch)"
    cur = torch.cuda.current_stream()
    side = _side_stream(cur.device)
    side.wait_stream(cur)
    with torch.cuda.stream(side):
        result = fn()

    def join():
        cur.wait_stream(side)
        for t in _tensors(result):
            t.record_stream(cur)
        return result
    return join


def branch_overlap(x):
    """template / search branches on two streams: inference on the device, fused execution"""
    return x.is_cuda and not torch.is_grad_enabled() and runtime.fused_enabled() and runtime.branch_overlap_enabled()
