"""Process-wide execution switches (read by the modules; no global state inside the native library)."""
import contextlib
import os

_FUSED = os.environ.get("O3D_FUSED", "1") != "0"


# wgmma 3xTF32 GEMM core for the point-wise layers: bit 0 = forward + dgrad, bit 1 = wgrad  (0 = exact-fp32 CUDA cores)
_TC = int(os.environ.get("O3D_TC", "3"))


# Lifted first layer of grouped stacks (include/o3d_b200.h o3d_lift_t): 1 = the grouped tensor is never built (default),
# 0 = materialising ball-query+group kernel followed by a GEMM over the grouped rows (round-1 path, kept as a cross-check)
_LIFT = os.environ.get("O3D_LIFT", "1") != "0"


def lift_enabled() -> bool:
    return _LIFT


def set_lift(flag: bool) -> None:
    global _LIFT
    _LIFT = bool(flag)


_SA_FUSED = os.environ.get("O3D_SA_FUSED", "1") != "0"


def sa_fused_enabled() -> bool:
    """eval-mode forward passes (no autograd) run every set-abstraction layer as ONE kernel (csrc/sa_fused.cu)"""
    return _SA_FUSED


def set_sa_fused(flag: bool) -> None:
    global _SA_FUSED
    _SA_FUSED = bool(flag)


_BRANCH_OVERLAP = os.environ.get("O3D_BRANCH_OVERLAP", "1") != "0"


def branch_overlap_enabled() -> bool:
    """inference: the template branch runs on a side stream next to the search branch (fused.run_ahead)"""
    return _BRANCH_OVERLAP


def set_branch_overlap(flag: bool) -> None:
    global _BRANCH_OVERLAP
    _BRANCH_OVERLAP = bool(flag)


# Inference with static weights (the tracking loop): eval-mode stacks pack their weights and fold their running BatchNorm
# statistics ONCE (o3d_stack_prepare) instead of per call.  Off by default; static_weights_scope() turns it on.
_STATIC_WEIGHTS = False

# Advanced by the engine once per training step.  Its Adam writes the parameters through a raw pointer, a graph replay bumps no
# tensor version, and the fused training forward writes the BatchNorm running statistics through pointers: none of these is
# visible in `Tensor._version`, so every static-weight cache entry also records the generation it was built in.
_WEIGHTS_GENERATION = 0


def weights_generation() -> int:
    return _WEIGHTS_GENERATION


def advance_weights_generation() -> None:
    global _WEIGHTS_GENERATION
    _WEIGHTS_GENERATION += 1


def static_weights() -> bool:
    return _STATIC_WEIGHTS


@contextlib.contextmanager
def static_weights_scope():
    """`with runtime.static_weights_scope():` — inference code whose weights do not change while it runs.

    The cached blocks are keyed by the identity and tensor version of every tensor they are computed from: the parameters and
    the running mean and variance of every BatchNorm that tracks them, so `load_state_dict` and other in-place updates rebuild
    them.  They also record the weights generation, which every `engine.TrainStep.step` / `FlatAdam.step` advances, so the
    first forward after a training step rebuilds them, whether or not a scope was open across the step."""
    global _STATIC_WEIGHTS
    old = _STATIC_WEIGHTS
    _STATIC_WEIGHTS = True
    try:
        yield
    finally:
        _STATIC_WEIGHTS = old


# Operand precision of the tensor-core forward GEMMs in inference (include/o3d_b200.h o3d_stack_t.precision): "fp32" = 3xTF32
# (default, fp32-grade), "bf16" = BF16 operands with FP32 accumulation.  Only inference_precision_scope() changes it.
PRECISIONS = ("fp32", "bf16")
_PRECISION = "fp32"


def inference_precision() -> str:
    return _PRECISION


def check_precision(precision) -> str:
    """`precision` if it is one of PRECISIONS, else a ValueError"""
    if precision not in PRECISIONS:
        raise ValueError(f"precision must be one of {PRECISIONS}, got {precision!r}")
    return precision


@contextlib.contextmanager
def inference_precision_scope(precision):
    """`with runtime.inference_precision_scope("bf16"):` — eval-mode forward passes without autograd run their tensor-core GEMMs
    (the fused SA layer and the pw_tc forward) on BF16 operands with FP32 accumulation.  A bf16 block is a prepared parameter
    block, so the scope also turns on static weights (static_weights_scope); its blocks are cached beside the fp32 ones.  A
    forward that needs a gradient, or a module in training mode, raises a RuntimeError inside a "bf16" scope.  Layers that run on
    the exact-fp32 CUDA-core kernels, and everything outside the MLP stacks (FPS, ball query, cross-correlation, box math), stay
    fp32.  "fp32" leaves every result as it is outside the scope."""
    global _PRECISION
    check_precision(precision)
    old = _PRECISION
    _PRECISION = precision
    try:
        if precision == "bf16":
            with static_weights_scope():
                yield
        else:
            yield
    finally:
        _PRECISION = old


# Operand precision of the tensor-core GEMMs of stacks in training mode (o3d_stack_t.precision 2): "fp32" = 3xTF32 (default),
# "bf16" = BF16 operands with FP32 accumulation in the forward, data-gradient and weight-gradient GEMMs.  Only
# training_precision_scope() changes it; engine.TrainStep(precision=...) opens it around its steps.
_TRAIN_PRECISION = "fp32"


def training_precision() -> str:
    return _TRAIN_PRECISION


@contextlib.contextmanager
def training_precision_scope(precision):
    """`with runtime.training_precision_scope("bf16"):` — MLP stacks in training mode run their tensor-core forward, dgrad and
    wgrad GEMMs on BF16 operands with FP32 accumulation (include/o3d_b200.h, o3d_stack_t.precision = 2).  Parameters, gradients,
    optimizer state, BatchNorm statistics, the stored layer outputs and every layer on the CUDA-core kernels stay fp32.
    Eval-mode stacks, with or without autograd, ignore the scope, so a validation inside it runs as it would outside.  "fp32"
    leaves every result as it is outside the scope."""
    global _TRAIN_PRECISION
    check_precision(precision)
    old = _TRAIN_PRECISION
    _TRAIN_PRECISION = precision
    try:
        yield
    finally:
        _TRAIN_PRECISION = old


# In-place accumulation of parameter gradients: a stack's backward ADDS its weight / bias / BatchNorm gradients straight into the
# parameters' existing `.grad` buffers (and returns no gradient for them) instead of materialising them and letting autograd's
# AccumulateGrad issue one elementwise add per parameter — ~130 launches per BAT step.  Only valid for `loss.backward()` onto
# pre-allocated `.grad` buffers (the engine's flat bucket); `torch.autograd.grad` callers must leave it off (default).
_GRAD_INPLACE = False


def grad_inplace() -> bool:
    return _GRAD_INPLACE


@contextlib.contextmanager
def grad_inplace_scope():
    global _GRAD_INPLACE
    old = _GRAD_INPLACE
    _GRAD_INPLACE = True
    try:
        yield
    finally:
        _GRAD_INPLACE = old


# (row count, plan threshold) pairs of the fused MLP stacks that run inside stack_rows_scope() (None outside one).
_STACK_ROWS = None


def recording_stack_rows() -> bool:
    return _STACK_ROWS is not None


def note_stack_rows(P, thresholds) -> None:
    """Record a stack forward of P rows whose kernel plan changes at the row counts `thresholds`."""
    if _STACK_ROWS is not None:
        _STACK_ROWS.update((int(P), int(t)) for t in thresholds)


@contextlib.contextmanager
def stack_rows_scope():
    """`with runtime.stack_rows_scope() as rows:` — `rows` (a set) collects, for every fused MLP stack forward run inside, its
    row count P paired with each row count at which that stack's kernel plan changes (include/o3d_b200.h,
    o3d_stack_plan_thresholds).  A caller that runs one network at several batch sizes reads from it which sizes share one
    kernel plan."""
    global _STACK_ROWS
    old = _STACK_ROWS
    _STACK_ROWS = set()
    try:
        yield _STACK_ROWS
    finally:
        _STACK_ROWS = old


def tc_level() -> int:
    return _TC


def set_tc(level) -> None:
    global _TC
    _TC = int(level)


def fused_enabled() -> bool:
    return _FUSED


def set_fused(flag: bool) -> None:
    global _FUSED
    _FUSED = bool(flag)


@contextlib.contextmanager
def composed_mode():
    """Run modules as the reference's op-by-op composition over the nine `_ext` kernels (cross-check path)."""
    global _FUSED
    old = _FUSED
    _FUSED = False
    try:
        yield
    finally:
        _FUSED = old


# ---- discrete-choice hook (parity tests only) -------------------------------------------------------------------
# The forward pass takes data-dependent DISCRETE decisions on computed values: the ball query of every set-abstraction layer
# (on input coordinates in the backbone, on VOTED coordinates in the RPN), BoxAwareXCorr's top-k over predicted box clouds, and
# M2-Track's arg-max point mask and motion state ("m2_segment", "m2_motion_state").  A neighbour that sits within fp32
# round-off of the radius / of the k-th distance can fall the other way on the GPU than in the CPU oracle, which changes
# downstream floats by O(1e-3) without any kernel being wrong.
# Parity tests install a hook that (a) records the product's own choice and (b) may substitute the oracle's, so that the
# float path is compared at 1e-4 with identical discrete choices.  hook(kind, info, compute) -> int32 tensor; `compute()`
# evaluates the product's choice.  None (the default) = no hook: the product path is unchanged.
CHOICE_HOOK = None


def choose(kind, info, compute):
    if CHOICE_HOOK is None:
        return compute()
    return CHOICE_HOOK(kind, info, compute)
