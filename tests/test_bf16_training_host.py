"""BF16 training precision without a GPU: o3d_stack_t.precision = 2 in the C ABI's planning and refusals, the runtime's training
precision scope and the precision code a stack gets from it, and the `precision` argument of TrainStep, the Trainer and the
command line."""
import ctypes
import os

import pytest

from open3dsot_b200 import _lib, fused, runtime
from open3dsot_b200.config import load_config
from open3dsot_b200.main import parse_config
from open3dsot_b200.trainer import Trainer, check_supported
from test_bf16_host import BF16_TILE, DUMMY, TF32_TILE, _stack_desc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CFG = os.path.join(ROOT, "cfgs", "BAT_Car.yaml")


def _sizes(d):
    L = _lib.lib()
    return L.o3d_stack_workspace_bytes(ctypes.byref(d), 0), L.o3d_stack_workspace_bytes(ctypes.byref(d), 1)


@pytest.mark.parametrize("widths, P, tiles", [
    # 64 -> 128 -> 256 at P = 4096: forward images 1 x 2 + 2 x 4, dgrad images 1 x 4 + 1 x 8 (channel tile x k-block)
    ([64, 128, 256], 4096, 22),
    # 128 -> 128 -> 128 at P = 65,536 (the fused narrow-layer backward): forward 1 x 4 twice, dgrad 1 x 4 twice
    ([128, 128, 128], 65536, 16),
    # a first layer with a ragged 4-channel tail (K0 = 132): its dgrad images cover the 128 tensor-core input channels only
    ([132, 128, 64], 4096, 5 + 4 + 4 + 2),
])
def test_bf16_training_plans_with_bf16_tiles(widths, P, tiles):
    fwd32, bwd32 = _sizes(_stack_desc(widths, P, precision=0, training=1))
    fwd16, bwd16 = _sizes(_stack_desc(widths, P, precision=2, training=1))
    assert fwd32 > 0 and bwd32 > 0
    assert fwd32 - fwd16 == tiles * (TF32_TILE - BF16_TILE)       # the weight images live in the forward workspace
    assert bwd16 == bwd32                                          # the backward workspace (partial tiles included) is fp32


def test_bf16_training_keeps_the_cuda_core_layers():
    # P < 128: every training layer on the exact-fp32 CUDA-core kernels, which have no tiles: the same plan in either precision
    assert _sizes(_stack_desc([64, 128, 256], 64, precision=2, training=1)) == _sizes(_stack_desc([64, 128, 256], 64, training=1))


def test_bf16_training_is_refused_in_eval_mode():
    L = _lib.lib()
    d = _stack_desc([64, 128, 256], 4096, precision=2, training=0)
    assert L.o3d_stack_prepared_bytes(ctypes.byref(d)) == -1
    assert _sizes(d) == (-1, -1)
    assert L.o3d_stack_prepare(ctypes.byref(d), DUMMY, None) < 0
    assert L.o3d_stack_forward(ctypes.byref(d), DUMMY, DUMMY, DUMMY, 0, None) < 0
    assert b"precision" in L.o3d_last_error()
    assert L.o3d_stack_backward(ctypes.byref(d), DUMMY, DUMMY, DUMMY, DUMMY, DUMMY, None, None) < 0
    d.precision = 3                                                # unknown precision, training or not
    for training in (0, 1):
        d.training = training
        assert _sizes(d) == (-1, -1)


def test_bf16_inference_precision_keeps_its_refusals():
    L = _lib.lib()
    d = _stack_desc([64, 128, 256], 4096, precision=1, training=1)
    assert _sizes(d) == (-1, -1)                                   # precision 1 does not plan a training stack
    assert L.o3d_stack_backward(ctypes.byref(d), DUMMY, DUMMY, DUMMY, DUMMY, DUMMY, None, None) < 0
    assert b"inference" in L.o3d_last_error()
    d.training = 0
    assert L.o3d_stack_backward(ctypes.byref(d), DUMMY, DUMMY, DUMMY, DUMMY, DUMMY, None, None) < 0
    assert b"inference" in L.o3d_last_error()
    assert _lib.PRECISION_BF16_TRAIN == 2


def test_training_precision_scope_validates_and_restores():
    assert runtime.training_precision() == "fp32"
    with runtime.training_precision_scope("bf16"):
        assert runtime.training_precision() == "bf16"
        assert runtime.inference_precision() == "fp32" and not runtime.static_weights()
        with runtime.training_precision_scope("fp32"):
            assert runtime.training_precision() == "fp32"
        assert runtime.training_precision() == "bf16"
    assert runtime.training_precision() == "fp32"
    for bad in ("fp16", "BF16", None):
        with pytest.raises(ValueError, match="precision"):
            with runtime.training_precision_scope(bad):
                pass
    assert runtime.training_precision() == "fp32"
    with pytest.raises(KeyError):                                  # restored when the body raises
        with runtime.training_precision_scope("bf16"):
            raise KeyError
    assert runtime.training_precision() == "fp32"


def test_stack_precision_code():
    code = fused._precision_code
    for training, need_grad in ((True, True), (True, False), (False, True), (False, False)):
        assert code(training, need_grad) == _lib.PRECISION_TF32X3
    with runtime.training_precision_scope("bf16"):
        assert code(True, True) == code(True, False) == _lib.PRECISION_BF16_TRAIN
        assert code(False, True) == _lib.PRECISION_TF32X3          # eval-mode stacks ignore the training scope
        assert code(False, False) == _lib.PRECISION_TF32X3
        with runtime.inference_precision_scope("bf16"):
            assert code(False, False) == _lib.PRECISION_BF16
            for training, need_grad in ((True, True), (True, False), (False, True)):
                with pytest.raises(RuntimeError, match="bf16 inference precision"):
                    code(training, need_grad)


@pytest.mark.parametrize("bad", ["fp16", "BF16", None, 2])
def test_train_step_and_trainer_refuse_unknown_precision(bad):
    from open3dsot_b200.engine import TrainStep
    with pytest.raises(ValueError, match="precision"):
        TrainStep(None, precision=bad)                             # checked before the model is looked at
    cfg = load_config(CFG)
    cfg.train_precision = bad
    with pytest.raises(ValueError, match="train_precision"):
        check_supported(cfg)
    with pytest.raises(ValueError, match="train_precision"):
        Trainer(None, cfg, [], [], "unused")


def test_command_line_takes_train_precision():
    assert parse_config(["--cfg", CFG]).train_precision == "fp32"
    cfg = parse_config(["--cfg", CFG, "--train_precision", "bf16"])
    assert cfg.train_precision == "bf16" and cfg.precision == "fp32"
    check_supported(cfg)
    check_supported(load_config(CFG))                              # a config without the key trains in fp32
    with pytest.raises(SystemExit):
        parse_config(["--cfg", CFG, "--train_precision", "fp16"])
    # --precision stays the inference precision of --test: training still refuses it, with or without --train_precision
    cfg = parse_config(["--cfg", CFG, "--train_precision", "bf16", "--precision", "bf16"])
    with pytest.raises(ValueError, match="precision: 'bf16' is for inference only"):
        check_supported(cfg)
    assert parse_config(["--cfg", CFG, "--test", "--train_precision", "bf16"]).test
