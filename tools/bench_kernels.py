"""Per-shape kernel micro-benchmarks at the UNet's real shapes (forward batch 8 = cond+uncond of 4
images at 512^2).  Each shape: 3 warm-ups, then N timed launches bracketed by CUDA events on the
launching stream with an L2 flush (256 MB write) between launches.  Prints one table row per shape
and a JSON blob (gpurun_out/kernels_<tag>.json).

  python tools/bench_kernels.py [tag] [gemm|attn|norm|conv_in|all] [--batch N] [--batch-invariant]

--batch-invariant runs every kernel in batch-invariant mode (ops.set_batch_invariant), so per-shape costs of the
two modes can be compared; --batch sets the forward batch (default 8).
"""
import json
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from instancediffusion_b200 import ops  # noqa: E402
from instancediffusion_b200.packing import pack_conv3x3, pack_conv3x3_taps, pack_geglu  # noqa: E402

dev = torch.device("cuda:0")
argv = [a for a in sys.argv[1:] if a != "--batch-invariant"]
B = 8
if "--batch" in argv:
    i = argv.index("--batch")
    B = int(argv[i + 1])
    del argv[i:i + 2]
tag = argv[0] if len(argv) > 0 else "run"
which = argv[1] if len(argv) > 1 else "all"
ops.set_batch_invariant("--batch-invariant" in sys.argv)
flush = torch.zeros(64 << 20, dtype=torch.int32, device=dev)  # 256 MB, read to evict L2 with clean lines


def timed(fn, iters=5):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        flush.sum()  # read 256 MB: L2 now holds clean lines of `flush` only (a write-flush would leave
        # 126 MB of dirty lines whose eviction is billed to the kernel under test)
        # keep the GPU busy (~150 us) while the CPU enqueues, so the events bracket pure device time
        torch.cuda._sleep(300000)
        s = torch.cuda.Event(enable_timing=True)
        e = torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e) * 1e-3)
    ts.sort()
    return ts[len(ts) // 2]


def rnd(*shape, scale=1.0):
    return (torch.randn(*shape, device=dev) * scale).half()


rows = []

# (label, count per forward, M, N, K, kind) -- kinds: lin, lin_res, geglu, conv (H, W, Cin)
L = [(4096, 320, 64), (1024, 640, 32), (256, 1280, 16), (64, 1280, 8)]
gemm_shapes = []
for (hw, C, res), nblk in zip(L[:3], (5, 5, 5)):
    M = B * hw
    gemm_shapes += [
        (f"qkv C{C}", 2 * nblk, M, 3 * C, C, "lin"),
        (f"attn-out/proj C{C}", 5 * nblk, M, C, C, "lin_res"),
        (f"geglu C{C}", 2 * nblk, M, 8 * C, C, "geglu"),
        (f"ff2 C{C}", 2 * nblk, M, C, 4 * C, "lin_res"),
    ]
gemm_shapes += [
    ("qkv C1280@8", 2, B * 64, 3840, 1280, "lin"), ("geglu C1280@8", 2, B * 64, 10240, 1280, "geglu"),
    ("ff2 C1280@8", 2, B * 64, 1280, 5120, "lin_res"),
    ("emb_all", 1, B, 20160, 1280, "lin"), ("ctx_kv_all", 0, B * 77, 24960, 768, "lin"),
]
conv_shapes = [
    ("conv 320->320 @64", 4, 64, 320, 320), ("conv 640->320 @64", 2, 64, 640, 320), ("conv 960->320 @64", 1, 64, 960, 320),
    ("conv 640->640 @64 (up)", 1, 64, 640, 640),
    ("conv 640->640 @32", 6, 32, 640, 640), ("conv 320->640 @32", 1, 32, 320, 640), ("conv 1280->640 @32", 1, 32, 1280, 640),
    ("conv 1920->640 @32", 1, 32, 1920, 640), ("conv 960->640 @32", 1, 32, 960, 640), ("conv 1280->1280 @32 (up)", 1, 32, 1280, 1280),
    ("conv 1280->1280 @16", 9, 16, 1280, 1280), ("conv 640->1280 @16", 1, 16, 640, 1280), ("conv 2560->1280 @16", 2, 16, 2560, 1280),
    ("conv 1920->1280 @16", 1, 16, 1920, 1280),
    ("conv 1280->1280 @8", 11, 8, 1280, 1280), ("conv 2560->1280 @8", 3, 8, 2560, 1280),
]

if which in ("all", "gemm"):
    print(f"{'shape':30s} {'cnt':>3s} {'M':>6s} {'N':>6s} {'K':>6s} {'us':>8s} {'TFLOP/s':>8s} {'GB/s':>8s}")
    for label, cnt, M, N, K, kind in gemm_shapes:
        a = rnd(M, K)
        w = rnd(N, K, scale=1 / math.sqrt(K))
        bias = torch.randn(N, device=dev)
        if kind == "geglu":
            wp, bp = pack_geglu(w, bias)
            out = torch.empty((M, N // 2), dtype=torch.float16, device=dev)
            fn = lambda: ops.gemm(a, wp, bp, geglu=True, out=out)
            nout = N // 2
        elif kind == "lin_res":
            res = rnd(M, N)
            out = torch.empty((M, N), dtype=torch.float16, device=dev)
            fn = lambda: ops.gemm(a, w, bias, residual=res, out=out)
            nout = N
        else:
            out = torch.empty((M, N), dtype=torch.float16, device=dev)
            fn = lambda: ops.gemm(a, w, bias, out=out)
            nout = N
        t = timed(fn)
        fl = 2.0 * M * N * K
        by = 2.0 * (M * K + N * K + M * nout * (2 if kind == "lin_res" else 1))
        rows.append(dict(kind="gemm", label=label, count=cnt, M=M, N=N, K=K, us=t * 1e6, tflops=fl / t / 1e12, gbs=by / t / 1e9))
        print(f"{label:30s} {cnt:3d} {M:6d} {N:6d} {K:6d} {t * 1e6:8.1f} {fl / t / 1e12:8.1f} {by / t / 1e9:8.0f}")
    for label, cnt, hw, cin, cout in conv_shapes:
        M = B * hw * hw
        a = rnd(M, cin)
        w = rnd(cout, 9 * cin, scale=1 / math.sqrt(9 * cin))
        bias = torch.randn(cout, device=dev)
        res = rnd(M, cout)
        out = torch.empty((M, cout), dtype=torch.float16, device=dev)
        fn = lambda: ops.gemm(a, w, bias, conv=(B, hw, hw, cin), residual=res, out=out)
        t = timed(fn)
        fl = 2.0 * M * cout * 9 * cin
        by = 2.0 * (M * cin + cout * 9 * cin + 2 * M * cout)
        rows.append(dict(kind="conv", label=label, count=cnt, M=M, N=cout, K=9 * cin, us=t * 1e6, tflops=fl / t / 1e12, gbs=by / t / 1e9))
        print(f"{label:30s} {cnt:3d} {M:6d} {cout:6d} {9 * cin:6d} {t * 1e6:8.1f} {fl / t / 1e12:8.1f} {by / t / 1e9:8.0f}")
    tot = sum(r["us"] * r["count"] for r in rows)
    fl = sum(r["us"] * r["count"] * r["tflops"] for r in rows)
    print(f"GEMM+conv per forward (count-weighted): {tot / 1e3:.2f} ms, {fl / tot:.1f} TFLOP/s average")
    # The epilogues the forward actually runs at the short-K levels (the rows above use plain / residual stand-ins
    # and stay as they are so that old and new numbers compare).  bound: the larger of FLOPs at 989 TFLOP/s and
    # bytes at 3.35 TB/s (H100 SXM data sheet), so x bound is how far a launch is from either roof.
    print(f"{'epilogue variant':30s} {'M':>6s} {'N':>6s} {'K':>6s} {'us':>8s} {'TFLOP/s':>8s} {'GB/s':>8s} {'x bound':>8s}")
    for hw, C in ((4096, 320), (1024, 640)):
        M = B * hw
        a = rnd(M, C)
        res = rnd(M, C)
        w = rnd(C, C, scale=1 / math.sqrt(C))
        bias = torch.randn(C, device=dev)
        _, st = ops.gemm(a, w, bias, residual=res, want_stats=True)
        ones = torch.ones(B, device=dev)
        gamma, beta = torch.ones(C, device=dev), torch.zeros(C, device=dev)
        fq = ops.fold_layernorm(torch.randn(3 * C, C, device=dev) / math.sqrt(C), None, gamma, beta, 1e-5)
        fg = ops.fold_layernorm(torch.randn(8 * C, C, device=dev) / math.sqrt(C), torch.randn(8 * C, device=dev),
                                gamma, beta, 1e-5, pack=pack_geglu)
        o3 = torch.empty((M, 3 * C), dtype=torch.float16, device=dev)
        o4 = torch.empty((M, 4 * C), dtype=torch.float16, device=dev)
        o1 = torch.empty((M, C), dtype=torch.float16, device=dev)
        wc = rnd(C, 9 * C, scale=1 / math.sqrt(9 * C))
        emb = rnd(B, C)
        cases = [  # label, fn, N, K, output columns, bytes beyond A, W and the output
            (f"qkv LN-fold C{C}", lambda: ops.gemm(a, fq.w, fq.bias, ln=(st, fq.colsum, fq.eps), out=o3), 3 * C, C, 3 * C, 0),
            (f"geglu LN-fold C{C}", lambda: ops.gemm(a, fg.w, fg.bias, geglu=True, ln=(st, fg.colsum, fg.eps), out=o4),
             8 * C, C, 4 * C, 0),
            (f"proj + stats C{C}", lambda: ops.gemm(a, w, bias, residual=res, out=o1, want_stats=True), C, C, C, 2 * M * C),
            (f"gated proj + stats C{C}", lambda: ops.gemm(a, w, bias, residual=res, gate_rows=ones, rows_per_batch=hw,
                                                          out=o1, want_stats=True), C, C, C, 2 * M * C),
            (f"conv + rowadd C{C}", lambda: ops.gemm(a, wc, bias, conv=(B, int(hw ** 0.5), int(hw ** 0.5), C), rowadd=emb,
                                                     out=o1), C, 9 * C, C, 0),
        ]
        for label, fn, N, K, nout, extra in cases:
            t = timed(fn)
            fl = 2.0 * M * N * K
            by = 2.0 * (M * min(K, C) + N * K + M * nout) + extra
            bound = max(fl / 989e12, by / 3.35e12)
            rows.append(dict(kind="gemm_variant", label=label, count=0, M=M, N=N, K=K, us=t * 1e6, tflops=fl / t / 1e12,
                             gbs=by / t / 1e9, bound_us=bound * 1e6))
            print(f"{label:30s} {M:6d} {N:6d} {K:6d} {t * 1e6:8.1f} {fl / t / 1e12:8.1f} {by / t / 1e9:8.0f} {t / bound:8.2f}")

if which in ("all", "attn"):
    print(f"\n{'attention':30s} {'cnt':>3s} {'Nq':>6s} {'Nkv':>6s} {'d':>4s} {'us':>8s} {'TFLOP/s':>8s}")
    for (hw, C, res), cnt in zip(L, (5, 5, 5, 1)):
        d = C // 8
        qkv = rnd(B * hw, 3 * C)
        okv = rnd(B * 184, 2 * C)
        ckv = rnd(B * 77, 2 * C)
        out = torch.empty((B * hw, C), dtype=torch.float16, device=dev)
        cases = [
            ("self", hw, 0, lambda: ops.attention(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], batch=B, heads=8, head_dim=d, nq=hw, n0=hw, scale=d ** -0.5, out=out)),
            ("gated", hw, 184, lambda: ops.attention(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], batch=B, heads=8, head_dim=d, nq=hw, n0=hw, scale=d ** -0.5, k1=okv[:, :C], v1=okv[:, C:], n1=184, kv1_batch=B, out=out)),
            ("cross", 77, 0, lambda: ops.attention(qkv[:, :C], ckv[:, :C], ckv[:, C:], batch=B, heads=8, head_dim=d, nq=hw, n0=77, scale=d ** -0.5, out=out)),
        ]
        for name, n0, n1, fn in cases:
            t = timed(fn)
            fl = 4.0 * B * 8 * hw * (n0 + n1) * d
            rows.append(dict(kind="attn", label=f"{name} N{hw} d{d}", count=cnt, us=t * 1e6, tflops=fl / t / 1e12))
            print(f"{name + f' N{hw}':30s} {cnt:3d} {hw:6d} {n0 + n1:6d} {d:4d} {t * 1e6:8.1f} {fl / t / 1e12:8.1f}")

if which in ("all", "norm"):
    print(f"\n{'norm / elementwise':30s} {'us':>8s} {'GB/s (4B/elt)':>14s}")
    # UNet shapes, then VAE decoder planes (the two largest at one image: 512 MB per batch-8 tensor)
    for hw, C in [(4096, 320), (4096, 640), (4096, 960), (1024, 640), (1024, 1280), (1024, 1920), (256, 1280), (256, 2560), (64, 1280), (64, 2560),
                  (4096, 512), (16384, 512), (65536, 256), (262144, 128)]:
        Bn = 1 if hw * C > (1 << 24) else B
        x = rnd(Bn * hw, C)
        g = torch.ones(C, device=dev)
        bb = torch.zeros(C, device=dev)
        out = torch.empty_like(x)
        t = timed(lambda: ops.groupnorm(x, g, bb, batch=Bn, hw=hw, silu=True, out=out))
        rows.append(dict(kind="groupnorm", label=f"gn {hw}x{C}", us=t * 1e6, gbs=4.0 * x.numel() / t / 1e9))
        print(f"{f'groupnorm {hw}x{C}':30s} {t * 1e6:8.1f} {4.0 * x.numel() / t / 1e9:14.0f}")
    for hw, C in [(4096, 320), (1024, 640), (256, 1280), (64, 1280)]:
        x = rnd(B * hw, C)
        g = torch.ones(C, device=dev)
        bb = torch.zeros(C, device=dev)
        out = torch.empty_like(x)
        t = timed(lambda: ops.layernorm(x, g, bb, out=out))
        rows.append(dict(kind="layernorm", label=f"ln {hw}x{C}", us=t * 1e6, gbs=4.0 * x.numel() / t / 1e9))
        print(f"{f'layernorm {hw}x{C}':30s} {t * 1e6:8.1f} {4.0 * x.numel() / t / 1e9:14.0f}")
    for hw, c1, c2 in [(64, 1280, 1280), (256, 1280, 1280), (256, 1280, 640), (1024, 1280, 640), (1024, 640, 640), (1024, 640, 320), (4096, 640, 320), (4096, 320, 320)]:
        h = rnd(B * hw, c1)
        sk = rnd(B * hw, c2)
        b1 = torch.ones(c1, device=dev)
        s = int(math.isqrt(hw))
        out = torch.empty((B * hw, c1 + c2), dtype=torch.float16, device=dev)
        t = timed(lambda: ops.scaleu_concat(h, sk, b1, 1.3, batch=B, height=s, width=s, out=out))
        by = 4.0 * (h.numel() + sk.numel())
        rows.append(dict(kind="scaleu", label=f"scaleu {hw} {c1}+{c2}", us=t * 1e6, gbs=by / t / 1e9))
        print(f"{f'scaleu {hw} {c1}+{c2}':30s} {t * 1e6:8.1f} {by / t / 1e9:14.0f}")

if which in ("all", "conv_in"):
    # The UNet input conv (4 -> 320, 3x3) as the model runs it, ops.conv_in_select, against the conv GEMM over a
    # 64-channel zero-padded NHWC copy of the latent that the model ran before.  Batches: one request (2), config 2
    # (8), a full engine bucket (32), a config 5 Multi-instance group (256) at 64x64, and config 4 (16 at 96x96, bf16).
    print(f"\n{'input conv':30s} {'select us':>10s} {'gemm us':>10s} {'rel_l2':>8s}")
    for nb, hw, dtype in ((2, 64, torch.float16), (8, 64, torch.float16), (32, 64, torch.float16),
                          (256, 64, torch.float16), (16, 96, torch.bfloat16)):
        with ops.storage(dtype):
            x = torch.randn(nb, 4, hw, hw, device=dev)
            w = torch.randn(320, 4, 3, 3, device=dev) * 0.2
            bias = torch.randn(320, device=dev) * 0.1
            wt = pack_conv3x3_taps(w.to(dtype))
            flags = torch.zeros(nb, dtype=torch.int32, device=dev)
            wpad = torch.zeros(320, 64, 3, 3, dtype=dtype, device=dev)
            wpad[:, :4] = w.to(dtype)
            wg = pack_conv3x3(wpad)
            x16 = torch.empty((nb * hw * hw, 64), dtype=dtype, device=dev)
            out = torch.empty((nb * hw * hw, 320), dtype=dtype, device=dev)
            out_g = torch.empty_like(out)
            sel = lambda: ops.conv_in_select(x, wt, bias, wt, bias, flags, out=out)
            gem = lambda: ops.gemm(ops.nchw_f32_to_nhwc_f16(x, 64, out=x16), wg, bias, conv=(nb, hw, hw, 64), out=out_g)
            ts, tg = timed(sel, iters=21), timed(gem, iters=21)
            rel = ((out.float() - out_g.float()).norm() / out_g.float().norm()).item()
        label = f"conv_in B{nb} {hw}x{hw} {str(dtype)[6:]}"
        rows.append(dict(kind="conv_in", label=label, us=ts * 1e6, gemm_us=tg * 1e6, rel_l2=rel))
        print(f"{label:30s} {ts * 1e6:10.1f} {tg * 1e6:10.1f} {rel:8.1e}")

os.makedirs("gpurun_out", exist_ok=True)
json.dump(rows, open(f"gpurun_out/kernels_{tag}.json", "w"), indent=1)
