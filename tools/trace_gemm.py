"""Per-CTA phase timeline of one GEMM launch (idiff_set_gemm_trace: 16 %globaltimer stamps per CTA).
Usage: python tools/trace_gemm.py [--mainloop] <shape> [...]

--mainloop launches each shape data-parallel at its usual tile width (IDIFF_GEMM_PLAN) and reports the SM clocks one
64-deep k-block of the mainloop takes, against the 4 * BN clocks the tensor cores need for it, and the operand
bytes per clock per SM that rate pulls from L2."""
import os
import subprocess
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
    "geglu320": lambda: (r(B * 4096, 320), r(2560, 320, sc=0.05), dict(geglu=True)),
    "ff2_320": lambda: (r(B * 4096, 1280), r(320, 1280, sc=0.03), dict(residual=r(B * 4096, 320))),
    "ff2_640": lambda: (r(B * 1024, 2560), r(640, 2560, sc=0.02), dict(residual=r(B * 1024, 640))),
    "conv1280": lambda: (r(B * 256, 1280), r(1280, 11520, sc=0.01), dict(conv=(B, 16, 16, 1280), residual=r(B * 256, 1280))),
    "conv1280_8": lambda: (r(B * 64, 1280), r(1280, 11520, sc=0.01), dict(conv=(B, 8, 8, 1280), residual=r(B * 64, 1280))),
    "ff2_1280_8": lambda: (r(B * 64, 5120), r(1280, 5120, sc=0.02), dict(residual=r(B * 64, 1280))),
    "conv320": lambda: (r(B * 4096, 320), r(320, 2880, sc=0.02), dict(conv=(B, 64, 64, 320), residual=r(B * 4096, 320))),
    "conv640": lambda: (r(B * 1024, 640), r(640, 5760, sc=0.015), dict(conv=(B, 32, 32, 640), residual=r(B * 1024, 640))),
}
# slots written by gemm2_kernel (gemm2.cu, idiff_set_gemm_trace): 1-3 the CTA's first epilogue tile, 4-6 its last
names = ["entry", "tile0 mainloop", "tile0 staged", "tile0 stored", "last mainloop", "last staged", "last stored",
         "exit"]


def tile_width(w, kw):
    """The tile width gemm2.cu plans for these N (GEGLU is always 256): the widest with no padded columns."""
    if kw.get("geglu"):
        return 256
    n = w.shape[0]
    return min((256, 192, 160, 128), key=lambda bn: (-(-n // bn) * bn, -bn))


def m_tiles(a, kw):
    if "conv" not in kw:
        return -(-a.shape[0] // 128)
    b, h, wd, _ = kw["conv"]  # choose_patch (gemm2.cu)
    pw = 1
    while pw * 2 <= 128 and wd % (pw * 2) == 0:
        pw *= 2
    ph = 1
    while pw * ph * 2 <= 128 and ph < h:
        ph *= 2
    pb = 128 // (pw * ph)
    return (wd // pw) * -(-h // ph) * -(-b // pb)


def mainloop_report(t, mhz, a, w, kw, bn):
    """Data-parallel launch: CTA c runs tiles c, c + G, ...  Per k-block time of the tiles after the first: the span
    between the first and the last tile's mainloop end over the tiles between, less the consumers' epilogue
    (mainloop end -> staged) that each of those spans contains."""
    G = t.shape[0]
    KB = -(-w.shape[1] // 64)
    T = m_tiles(a, kw) * -(-w.shape[0] // bn)
    n_c = torch.tensor([len(range(c, T, G)) for c in range(G)])
    clk = lambda ns: ns.float() * mhz / 1e3
    need = 4.0 * bn
    stage = 16384 + 128 * bn
    if (n_c >= 2).any():
        m = n_c >= 2
        per_tile = clk(t[m, 4] - t[m, 1]) / (n_c[m] - 1)
        epi = clk(t[m, 2] - t[m, 1])
        kb = ((per_tile - epi) / KB).median().item()
        kb_all = (per_tile / KB).median().item()
        print(f"   mainloop: BN {bn}, {KB} k-blocks/tile, {T} tiles on {G} CTAs; steady-state {kb:.0f} clk/k-block "
              f"({kb / need:.2f}x the tensor cores' {need:.0f}), {stage / kb:.1f} B/clk/SM from L2; "
              f"with the consumers' epilogue spread over the k-blocks {kb_all:.0f} clk ({kb_all / need:.2f}x)")
    else:
        kb = (clk(t[:, 1] - t[:, 0]) / KB).median().item()
        print(f"   mainloop: BN {bn}, {KB} k-blocks/tile, {T} tiles on {G} CTAs (one each); entry -> mainloop end "
              f"{kb:.0f} clk/k-block ({kb / need:.2f}x the tensor cores' {need:.0f}), {stage / kb:.1f} B/clk/SM from L2")


args = sys.argv[1:]
mainloop = "--mainloop" in args
args = [x for x in args if x != "--mainloop"]
print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv"],
                     capture_output=True, text=True).stdout.strip())
lib = _lib.load()
trace = torch.zeros(256 * 16, dtype=torch.int64, device=dev)
for name in args:
    a, w, kw = shapes[name]()
    bn = tile_width(w, kw)
    if mainloop:
        os.environ["IDIFF_GEMM_PLAN"] = f"{bn},0"
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
    if mainloop:
        mainloop_report(t, mhz.item(), a, w, kw, bn)
