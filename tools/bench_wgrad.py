"""The 3xTF32 weight-gradient GEMMs, timed alone through the C ABI with CUDA events at the BAT-Car batch-48 shapes:
o3d_pw_wgrad_tc2 / o3d_pw_wgrad_tc_lift (pw_wgrad_tc_kernel + wgrad_reduce_kernel) at the wide layers, and the fused
narrow-layer backward o3d_pw_bwd_tc (pw_bwd_tc_kernel: data and weight gradient in one pass) at the shapes of
tools/bench_fused_backward.py.  Inputs are seeded on the device (bench_fused_backward.Layer).

Per shape: time per call, the algorithmic bytes (what the call has to move at least once: dY's streams, the layer input, and
for the fused kernel the data gradient written), the tensor-core work (3 TF32 MMAs per product, 3xTF32), and both as a share
of the H100 SXM data sheet's 3.35 TB/s and 495 dense TF32 TFLOP/s; "binds" names the roof with the larger share.

  --lib PATH   time this build of libo3d_b200.so; give it more than once to time several builds in one process, alternating
               per shape (default: the in-tree library)
  --dump DIR   after timing, run each call once more from zeroed outputs and write dW (and the fused kernel's data gradient
               and BatchNorm-backward sums) as .npy under DIR/<build index>/
usage: python tools/bench_wgrad.py [--iters 20] [--lib PATH ...] [--dump DIR]"""
import argparse
import ctypes
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np
import torch

from open3dsot_b200 import _lib
from bench_fused_backward import SHAPES as FUSED_SHAPES, Layer, time_ms

HBM_GBS = 3350.0
TF32_TFLOPS = 495.0
# name, P, Cout (dY channels), Cin (layer input channels), pooling group of dY (0 = dense), lifted input
WGRAD_SHAPES = [
    ("SA2 layer 2, search", 48 * 256 * 32, 256, 128, 32, False),
    ("SA2 layer 2, template", 48 * 128 * 32, 256, 128, 32, False),
    ("SA3 layer 1, search", 48 * 128 * 32, 256, 256, 0, True),
    ("SA3 layer 1, template", 48 * 64 * 32, 256, 256, 0, True),
    ("SA3 layer 2, search", 48 * 128 * 32, 256, 256, 32, False),
    ("SA3 layer 2, template", 48 * 64 * 32, 256, 256, 32, False),
]


def load(path):
    """A CDLL of the build at `path`, with the package's prototypes bound (the package's own handle is left untouched)."""
    saved_path, saved = _lib.LIB_PATH, _lib._lib
    try:
        _lib.LIB_PATH, _lib._lib = os.path.abspath(path), None
        return _lib.lib()
    finally:
        _lib.LIB_PATH, _lib._lib = saved_path, saved


def use(L):
    _lib._lib = L     # Layer's calls go through _lib.lib()


def _p(t):
    return ctypes.c_void_p(0 if t is None else t.data_ptr())


class WgradLayer(Layer):
    def wgrad(self):
        L, st = _lib.lib(), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        if self.lifted:
            rc = L.o3d_pw_wgrad_tc_lift(*self._dy(), ctypes.byref(self.lf), _p(self.gidx), _p(self.scale), _p(self.shift), 1,
                                        self.P, self.cout, self.cin, _p(self.dw), self.cin, _p(self.part), self.part.numel(), st)
        else:
            rc = L.o3d_pw_wgrad_tc2(*self._dy(), _p(self.x), self.cin, _p(self.scale), _p(self.shift), 1, self.P, self.cout,
                                    self.cin, _p(self.dw), self.cin, _p(self.part), self.part.numel(), st)
        assert rc == 0, L.o3d_last_error()

    def wgrad_bytes(self):
        P, co, ci = self.P, self.cout, self.cin
        dy = (2 * (P // self.S) * co if self.S else P * co) + P * co          # g (or dpool + sel) and y
        xin = P * 5 + self.z.numel() if self.lifted else P * ci               # gidx, s and z once, or x
        return 4 * (dy + xin + co * ci)                                        # + dW


def roofs(nbytes, mma_flops, ms):
    hbm = nbytes / (ms * 1e-3) / (HBM_GBS * 1e9)
    tc = mma_flops / (ms * 1e-3) / (TF32_TFLOPS * 1e12)
    return hbm, tc, ("HBM" if hbm >= tc else "TF32")


def device_line():
    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "power limit / clocks not available"
    return f"{name}; {q}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--lib", action="append", default=None, help="libo3d_b200.so to time (repeatable)")
    ap.add_argument("--dump", default=None, help="directory for the .npy outputs")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    libs = [load(p) for p in a.lib] if a.lib else [_lib.lib()]
    names = a.lib if a.lib else [_lib.LIB_PATH]
    print(f"# {device_line()}")
    print(f"# times per call (CUDA events, {a.iters} calls after 3 warm-up calls); shares of {HBM_GBS:.0f} GB/s and "
          f"{TF32_TFLOPS:.0f} TFLOP/s (3 TF32 MMAs per product)")
    for i, n in enumerate(names):
        print(f"# build {i}: {n}")
    hdr = f"# {'call':14s} {'layer':24s} {'P':>7s} {'Cout':>4s} {'Cin':>4s} {'MB':>6s} {'MMA GF':>7s}"
    for i in range(len(libs)):
        hdr += f" {f'b{i} ms':>8s} {f'b{i} HBM':>7s} {f'b{i} TC':>6s} {'binds':>5s}"
    print(hdr)
    rows = [("wgrad", s) for s in WGRAD_SHAPES] + [("fused bwd", s) for s in FUSED_SHAPES[:6]]
    for kind, (label, P, co, ci, S, lifted) in rows:
        use(libs[0])
        lay = WgradLayer(P, co, ci, S, lifted)
        fn = lay.wgrad if kind == "wgrad" else lay.fused
        nb = lay.wgrad_bytes() if kind == "wgrad" else lay.algorithmic_bytes()
        flops = 3 * 2.0 * P * co * ci * (1 if kind == "wgrad" else 2)
        line = f"  {kind:14s} {label:24s} {P:7d} {co:4d} {ci:4d} {nb / 1e6:6.1f} {flops / 1e9:7.1f}"
        for L in libs:
            use(L)
            ms = time_ms(fn, a.iters)
            hbm, tc, b = roofs(nb, flops, ms)
            line += f" {ms:8.3f} {hbm:7.2f} {tc:6.2f} {b:>5s}"
        print(line, flush=True)
        if a.dump:
            tag = f"{kind.replace(' ', '_')}_{label.replace(', ', '_').replace(' ', '_')}"
            for i, L in enumerate(libs):
                use(L)
                d = os.path.join(a.dump, str(i))
                os.makedirs(d, exist_ok=True)
                lay.dw.zero_()
                lay.out.zero_()
                lay.s12.zero_()
                fn()
                torch.cuda.synchronize()
                np.save(os.path.join(d, f"{tag}_dw.npy"), lay.dw.cpu().numpy())
                if kind != "wgrad":
                    np.save(os.path.join(d, f"{tag}_dx.npy"), lay.out.cpu().numpy())
                    np.save(os.path.join(d, f"{tag}_bnsums.npy"), lay.s12.cpu().numpy())
        del lay, fn
        torch.cuda.empty_cache()
    use(libs[0])


if __name__ == "__main__":
    main()
