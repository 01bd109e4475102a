"""BF16 inference precision without a GPU: the C ABI's refusals and prepared-block sizes for o3d_stack_t.precision = 0 / 1, the
`precision` argument of the trackers and of both command lines, and the trainer refusing bf16."""
import ctypes
import os

import pytest

from open3dsot_b200 import _lib, runtime
from open3dsot_b200.config import load_config
from open3dsot_b200.main import parse_config
from open3dsot_b200.track import parse_args as track_args
from open3dsot_b200.trainer import check_supported
from test_cabi import _sa_desc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TF32_TILE, BF16_TILE = 2 * 128 * 32 * 4, 128 * 32 * 2     # one 128-channel x 32-k weight tile: TF32 hi | lo, one bf16 image
DUMMY = ctypes.c_void_p(16)                               # never dereferenced by the checks and planning entry points


def _stack_desc(widths, P, precision=0, training=0):
    d = _lib.StackDesc()
    d.n_layers, d.P, d.K0, d.S, d.training, d.use_tc, d.precision = len(widths) - 1, P, widths[0], 0, training, 3, precision
    for l, (cin, cout) in enumerate(zip(widths[:-1], widths[1:])):
        d.cin[l], d.cout[l], d.relu[l], d.has_bn[l] = cin, cout, 1, 1
        d.weight[l] = d.gamma[l] = d.beta[l] = d.running_mean[l] = d.running_var[l] = DUMMY
    return d


def test_stack_forward_refuses_bf16_outside_prepared_inference():
    L = _lib.lib()
    d = _stack_desc([64, 128, 256], 4096, precision=1)
    assert L.o3d_stack_forward(ctypes.byref(d), DUMMY, DUMMY, DUMMY, 0, None) < 0               # no prepared block
    assert b"prepared" in L.o3d_last_error()
    d.prepared = DUMMY
    assert L.o3d_stack_forward(ctypes.byref(d), DUMMY, DUMMY, DUMMY, 1, None) < 0               # keep_for_backward
    assert b"precision" in L.o3d_last_error()
    d.training = 1
    assert L.o3d_stack_forward(ctypes.byref(d), DUMMY, DUMMY, DUMMY, 0, None) < 0               # training
    assert b"precision" in L.o3d_last_error()
    assert L.o3d_stack_prepared_bytes(ctypes.byref(d)) == -1
    assert L.o3d_stack_prepare(ctypes.byref(d), DUMMY, None) < 0
    d.training, d.precision = 0, 2                                                               # unknown precision
    assert L.o3d_stack_prepared_bytes(ctypes.byref(d)) == -1
    d.precision = 1
    assert L.o3d_stack_backward(ctypes.byref(d), DUMMY, DUMMY, DUMMY, DUMMY, DUMMY, None, None) < 0
    assert b"inference" in L.o3d_last_error()


def test_stack_prepared_block_holds_bf16_tiles():
    L = _lib.lib()
    # 64 -> 128 -> 256 at P = 4096: both layers on the tensor cores, 1 x 2 and 2 x 4 (channel tile x k-block) forward tiles
    fp32 = L.o3d_stack_prepared_bytes(ctypes.byref(_stack_desc([64, 128, 256], 4096)))
    bf16 = L.o3d_stack_prepared_bytes(ctypes.byref(_stack_desc([64, 128, 256], 4096, precision=1)))
    assert fp32 > 0 and fp32 - bf16 == 10 * (TF32_TILE - BF16_TILE)
    # P < 16: every layer on the exact-fp32 CUDA-core kernel, which has no tiles: the same block in either precision
    small = [L.o3d_stack_prepared_bytes(ctypes.byref(_stack_desc([64, 128, 256], 8, precision=p))) for p in (0, 1)]
    assert small[0] == small[1] > 0
    # zero-initialised descriptors keep the 3xTF32 default
    assert _lib.StackDesc().precision == _lib.PRECISION_TF32X3 == 0


def test_sa_fused_block_holds_bf16_tiles_and_refuses_training():
    L = _lib.lib()
    d = _sa_desc(256, [256, 256, 256])                                           # 48 tiles
    fp32 = L.o3d_sa_fused_prepared_bytes(ctypes.byref(d))
    d.precision = 1
    bf16 = L.o3d_sa_fused_prepared_bytes(ctypes.byref(d))
    assert fp32 - bf16 == 48 * (TF32_TILE - BF16_TILE)
    d.training = 1
    assert L.o3d_sa_fused_prepared_bytes(ctypes.byref(d)) == -1
    assert L.o3d_sa_fused_prepare(ctypes.byref(d), DUMMY, None) < 0
    assert L.o3d_sa_fused_forward(ctypes.byref(d), DUMMY, DUMMY, DUMMY, DUMMY, 256, 1, 64, 32, 0.3, 32, 0, DUMMY, 256, None,
                                  None) < 0


def test_precision_scope_validates_and_restores():
    assert runtime.inference_precision() == "fp32" and not runtime.static_weights()
    with runtime.inference_precision_scope("bf16"):
        assert runtime.inference_precision() == "bf16" and runtime.static_weights()
        with runtime.inference_precision_scope("fp32"):
            assert runtime.inference_precision() == "fp32"
        assert runtime.inference_precision() == "bf16"
    assert runtime.inference_precision() == "fp32" and not runtime.static_weights()
    with pytest.raises(ValueError, match="precision"):
        with runtime.inference_precision_scope("fp16"):
            pass


@pytest.mark.parametrize("bad", ["fp16", "BF16", None, 1])
def test_trackers_refuse_unknown_precision(bad):
    from open3dsot_b200.tracking.batched_tracker import BatchedDeviceTracker
    from open3dsot_b200.tracking.device_tracker import DeviceTracker
    from open3dsot_b200.tracking.evaluate import evaluate_batched, evaluate_sharded
    from open3dsot_b200.tracking.multi_tracker import MultiTargetTracker, track_feeds, track_stream
    # the precision is checked before the model or the data is looked at
    calls = [lambda: DeviceTracker(None, 100, precision=bad), lambda: BatchedDeviceTracker(None, [], 1, precision=bad),
             lambda: MultiTargetTracker(None, 100, 4, precision=bad), lambda: evaluate_batched(None, [], precision=bad),
             lambda: evaluate_sharded(None, [], precision=bad), lambda: track_stream(None, [], {}, {}, 4, precision=bad),
             lambda: track_feeds(None, [], 1, 4, precision=bad)]
    for call in calls:
        with pytest.raises(ValueError, match="precision"):
            call()


def test_command_lines_take_precision():
    base = ["--cfg", os.path.join(ROOT, "cfgs", "BAT_Car.yaml")]
    assert track_args(base + ["--path", "x"]).precision == "fp32"
    assert track_args(base + ["--path", "x", "--precision", "bf16"]).precision == "bf16"
    assert parse_config(base).precision == "fp32"
    assert parse_config(base + ["--test", "--precision", "bf16"]).precision == "bf16"
    with pytest.raises(SystemExit):
        track_args(base + ["--path", "x", "--precision", "fp16"])
    with pytest.raises(SystemExit):
        parse_config(base + ["--test", "--precision", "fp16"])


def test_training_refuses_bf16():
    cfg = parse_config(["--cfg", os.path.join(ROOT, "cfgs", "BAT_Car.yaml"), "--precision", "bf16"])
    with pytest.raises(ValueError, match="precision: 'bf16' is for inference only"):
        check_supported(cfg)
    check_supported(load_config(os.path.join(ROOT, "cfgs", "BAT_Car.yaml")))
