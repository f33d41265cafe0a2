"""Per-CTA phase timeline of one GEMM launch (idiff_set_gemm_trace: 16 %globaltimer stamps per CTA).
Usage: python tools/trace_gemm.py <shape> [...]"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from instancediffusion_b200 import _lib, ops

dev = torch.device("cuda:0")
B = 8
r = lambda *s, sc=1.0: (torch.randn(*s, device=dev) * sc).half()
shapes = {
    "proj1280": lambda: (r(B * 256, 1280), r(1280, 1280, sc=0.03), dict(residual=r(B * 256, 1280))),
    "proj320": lambda: (r(B * 4096, 320), r(320, 320, sc=0.05), dict(residual=r(B * 4096, 320))),
    "qkv320": lambda: (r(B * 4096, 320), r(960, 320, sc=0.05), dict()),
    "ff2_640": lambda: (r(B * 1024, 2560), r(640, 2560, sc=0.02), dict(residual=r(B * 1024, 640))),
    "conv1280": lambda: (r(B * 256, 1280), r(1280, 11520, sc=0.01), dict(conv=(B, 16, 16, 1280), residual=r(B * 256, 1280))),
    "conv1280_8": lambda: (r(B * 64, 1280), r(1280, 11520, sc=0.01), dict(conv=(B, 8, 8, 1280), residual=r(B * 64, 1280))),
    "ff2_1280_8": lambda: (r(B * 64, 5120), r(1280, 5120, sc=0.02), dict(residual=r(B * 64, 1280))),
    "conv320": lambda: (r(B * 4096, 320), r(320, 2880, sc=0.02), dict(conv=(B, 64, 64, 320), residual=r(B * 4096, 320))),
}
# slots written by gemm2_kernel (gemm2.cu, idiff_set_gemm_trace): 1-3 the CTA's first epilogue tile, 4-6 its last
names = ["entry", "tile0 mainloop", "tile0 staged", "tile0 stored", "last mainloop", "last staged", "last stored",
         "exit"]
lib = _lib.load()
trace = torch.zeros(256 * 16, dtype=torch.int64, device=dev)
for name in sys.argv[1:]:
    a, w, kw = shapes[name]()
    bias = torch.randn(w.shape[0], device=dev)
    for _ in range(3):
        ops.gemm(a, w, bias, **kw)
    torch.cuda.synchronize()
    trace.zero_()
    for _ in range(200):  # keep the GPU busy so the traced launch runs at load clocks
        ops.gemm(a, w, bias, **kw)
    lib.idiff_set_gemm_trace(trace.data_ptr())
    ops.gemm(a, w, bias, **kw)
    torch.cuda.synchronize()
    lib.idiff_set_gemm_trace(None)
    t = trace.view(256, 16).cpu()
    t = t[t[:, 0] > 0]
    t0 = t[:, 0].min()
    rel = (t - t0).float() / 1e3  # us
    mhz = ((t[:, 13] - t[:, 12]).float() / (t[:, 7] - t[:, 0]).float().clamp(min=1) * 1e3).median()
    print(f"== {name}: {t.shape[0]} CTAs, kernel span {rel[:, 7].max():.1f} us, SM clock during kernel ~{mhz:.0f} MHz")
    for i, n in enumerate(names):
        col = rel[:, i][t[:, i] > 0]
        if col.numel():
            print(f"   {n:16s} min {col.min():7.2f}  median {col.median():7.2f}  max {col.max():7.2f} us")
