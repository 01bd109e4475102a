"""Both gradients of one narrow layer, timed alone through the C ABI with CUDA events: the fused backward kernel
(o3d_pw_bwd_tc: dgrad and weight gradient in one pass over the operands) against the two-kernel pair it replaces
(o3d_pw_dgrad_tc(_lift), then o3d_pw_wgrad_tc2 / o3d_pw_wgrad_tc_lift), at the BAT-Car layers the fused path takes and
around the crossover P_FUSED_BWD (csrc/stack.cu).  Prints one row per shape: times, the algorithmic bytes (what the layer's
backward has to move at least once: dY's streams, the layer input, the data gradient written) and their rate as a share of
the H100 SXM data sheet's 3.35 TB/s.
usage: python tools/bench_fused_backward.py [--iters 20]"""
import argparse
import ctypes
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from open3dsot_b200 import _lib

HBM_GBS = 3350.0
# name, P, Cout (dY channels), Cin (layer input channels), pooling group of dY (0 = dense), lifted input
SHAPES = [
    ("SA1 layer 1, search", 48 * 512 * 32, 64, 64, 0, True),
    ("SA1 layer 1, template", 48 * 256 * 32, 64, 64, 0, True),
    ("SA1 layer 2, search", 48 * 512 * 32, 128, 64, 32, False),
    ("SA1 layer 2, template", 48 * 256 * 32, 128, 64, 32, False),
    ("SA2 layer 1, search", 48 * 256 * 32, 128, 128, 0, True),
    ("SA2 layer 1, template", 48 * 128 * 32, 128, 128, 0, True),
] + [(f"dense 128 -> 128, P = {p}", p, 128, 128, 0, False) for p in (16384, 32768, 65536, 131072)] \
  + [(f"pooled 128 -> 64, P = {p}", p, 128, 64, 32, False) for p in (16384, 32768, 65536, 131072)]


def _p(t):
    return ctypes.c_void_p(0 if t is None else t.data_ptr())


class Layer:
    """Seeded inputs of one layer's backward: dY = a * g + b + cc * y (g dense, or pooled: dpool[p / S] where sel == p % S),
    layer input X = relu(bn(x)) or the lifted Y0 = relu(bn(z[gidx] + s . u)), weight W [Cout, Cin] as its pre-tiled
    transposed image."""

    def __init__(self, P, cout, cin, S, lifted, seed=0):
        g = torch.Generator(device="cuda").manual_seed(seed)
        rn = lambda *shape: torch.randn(*shape, generator=g, device="cuda")   # noqa: E731
        self.P, self.cout, self.cin, self.S, self.lifted = P, cout, cin, S, lifted
        self.g = None if S else rn(P, cout)
        self.dpool = rn(P // S, cout) if S else None
        self.sel = torch.randint(0, S, (P // S, cout), generator=g, device="cuda", dtype=torch.int32) if S else None
        self.y = rn(P, cout)
        self.a, self.b, self.cc = rn(cout), 0.1 * rn(cout), 0.1 * rn(cout)
        self.scale, self.shift = 0.5 + torch.rand(cin, generator=g, device="cuda"), 0.2 * rn(cin)
        W = rn(cout, cin) / cin ** 0.5
        L = _lib.lib()
        self.tiles = torch.empty(L.o3d_pw_tc_wtile_bytes(cin, cout), dtype=torch.uint8, device="cuda")
        wt = W.t().contiguous()
        assert L.o3d_pw_tc_pretile(_p(wt), cout, cin, cout, _p(self.tiles), None) == 0
        torch.cuda.synchronize()
        self.x = self.z = self.gidx = self.s = self.u = self.lf = None
        if lifted:
            rows = max(P // 32, 1)
            self.z = rn(rows, cin)
            self.gidx = torch.randint(0, rows, (P,), generator=g, device="cuda", dtype=torch.int32)
            self.s = rn(P, 4)
            self.s[:, 3] = 0
            self.u = 0.5 * rn(4, cin)
            self.lf = _lib.LiftDesc()
            self.lf.z, self.lf.ldz, self.lf.s, self.lf.u = self.z.data_ptr(), cin, self.s.data_ptr(), self.u.data_ptr()
        else:
            self.x = rn(P, cin)
        self.part = torch.empty(L.o3d_pw_wgrad_tc2_workspace_floats(), device="cuda")
        self.out = torch.empty(P, cin, device="cuda")
        self.s12 = torch.zeros(2, cin, dtype=torch.float64, device="cuda")
        self.dw = torch.zeros(cout, cin, device="cuda")

    def _dy(self):
        return (_p(self.g), self.cout, _p(self.y), self.cout, _p(self.a), _p(self.b), _p(self.cc), _p(self.dpool), _p(self.sel),
                self.S, self.cout)

    def two_kernel(self):
        L, st = _lib.lib(), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        s1, s2 = _p(self.s12[0]), _p(self.s12[1])
        if self.lifted:
            lf = ctypes.byref(self.lf)
            rc = L.o3d_pw_dgrad_tc_lift(*self._dy(), _p(self.tiles), self.P, self.cout, self.cin, _p(self.out), self.cin, lf,
                                        _p(self.gidx), _p(self.scale), _p(self.shift), 1, s1, s2, st)
            rc = rc or L.o3d_pw_wgrad_tc_lift(*self._dy(), lf, _p(self.gidx), _p(self.scale), _p(self.shift), 1, self.P, self.cout,
                                              self.cin, _p(self.dw), self.cin, _p(self.part), self.part.numel(), st)
        else:
            rc = L.o3d_pw_dgrad_tc(*self._dy(), _p(self.tiles), self.P, self.cout, self.cin, _p(self.out), self.cin, _p(self.x),
                                   self.cin, _p(self.scale), _p(self.shift), 1, s1, s2, st)
            rc = rc or L.o3d_pw_wgrad_tc2(*self._dy(), _p(self.x), self.cin, _p(self.scale), _p(self.shift), 1, self.P, self.cout,
                                          self.cin, _p(self.dw), self.cin, _p(self.part), self.part.numel(), st)
        assert rc == 0, L.o3d_last_error()

    def fused(self):
        L, st = _lib.lib(), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        rc = L.o3d_pw_bwd_tc(*self._dy(), _p(self.tiles), _p(self.x), ctypes.byref(self.lf) if self.lifted else None,
                             _p(self.gidx), _p(self.scale), _p(self.shift), 1, self.P, self.cout, self.cin, _p(self.out),
                             _p(self.s12[0]), _p(self.s12[1]), _p(self.dw), self.cin, _p(self.part), self.part.numel(), st)
        assert rc == 0, L.o3d_last_error()

    def algorithmic_bytes(self):
        P, co, ci = self.P, self.cout, self.cin
        dy = (2 * (P // self.S) * co if self.S else P * co) + P * co          # g (or dpool + sel) and y
        xin = P * 5 if self.lifted else P * ci                                 # gidx and s (z rows stay in L2), or x
        return 4 * (dy + xin + P * ci)                                         # + the data gradient written


def time_ms(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    name = torch.cuda.get_device_name()
    print(f"# {name}; times per call (CUDA events, {a.iters} calls after 3 warm-up calls); GB/s and share of {HBM_GBS:.0f} GB/s "
          f"from the algorithmic bytes")
    print(f"# {'layer':32s} {'P':>8s} {'Cout':>4s} {'Cin':>4s} {'MB':>7s} {'2-kernel ms':>11s} {'fused ms':>9s} {'speed-up':>8s} "
          f"{'2-kernel GB/s':>13s} {'fused GB/s':>10s} {'fused share':>11s}")
    for label, P, co, ci, S, lifted in SHAPES:
        lay = Layer(P, co, ci, S, lifted)
        t2 = time_ms(lay.two_kernel, a.iters)
        tf = time_ms(lay.fused, a.iters)
        nb = lay.algorithmic_bytes()
        print(f"  {label:32s} {P:8d} {co:4d} {ci:4d} {nb / 1e6:7.1f} {t2:11.3f} {tf:9.3f} {t2 / tf:8.2f} {nb / t2 / 1e6:13.0f} "
              f"{nb / tf / 1e6:10.0f} {nb / tf / 1e6 / HBM_GBS:11.2f}", flush=True)
        del lay
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
