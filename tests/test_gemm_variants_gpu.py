"""The compiled-in GEMM epilogue variants (gemm2.cu EPI_*): each feature set the UNet launches -- no bias, bias,
LayerNorm fold (plain and GEGLU), residual with and without row statistics (plain and per-image gated), conv3x3
with a per-image row-add and conv3x3 with a residual -- against torch fp32 on the same 16-bit inputs, data-parallel
and stream-K, at M < 128 and M not a multiple of 128, with strided outputs between sentinels, conv patches clipped
by the image, a second launch bitwise equal to the first, and a CUDA-graph replay."""
import math
import os

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

SENTINEL = -7.0  # exactly representable in fp16 and bf16
TOL = {"fp16": 1.0, "bf16": 8.0}


@pytest.fixture(autouse=True, params=["fp16", "bf16"])
def storage(request):
    from instancediffusion_b200 import ops
    ops.set_storage_dtype(torch.bfloat16 if request.param == "bf16" else torch.float16)
    yield request.param
    ops.set_storage_dtype(torch.float16)


@pytest.fixture
def plan():
    def set_plan(bn, sk):
        os.environ["IDIFF_GEMM_PLAN"] = f"{bn},{int(sk)}"
    yield set_plan
    os.environ.pop("IDIFF_GEMM_PLAN", None)


def _ops():
    from instancediffusion_b200 import ops
    return ops


def _rand(shape, dev, scale=1.0, seed=0, half=True):
    g = torch.Generator(device="cpu").manual_seed(seed)
    t = (torch.randn(shape, generator=g) * scale).to(dev)
    return t.to(_ops().HALF) if half else t


def _close(got, ref, storage, what, tol=3e-3):
    got, ref = got.float(), ref.float()
    assert torch.isfinite(got).all(), f"{what}: non-finite output"
    err = (got - ref).abs()
    bad = err > TOL[storage] * tol * (1.0 + ref.abs())
    assert not bad.any(), f"{what}: max err {err.max().item():.3e}, {int(bad.sum())}/{bad.numel()} bad"


def _strided_out(M, N, dev):
    """An [M, N] view at a row and column offset of a sentinel-filled buffer, and a check of its surroundings."""
    buf = torch.full((M + 11, N + 48), SENTINEL, dtype=_ops().HALF, device=dev)
    out = buf[3:3 + M, 16:16 + N]

    def untouched():
        mask = torch.ones_like(buf, dtype=torch.bool)
        mask[3:3 + M, 16:16 + N] = False
        return bool((buf[mask] == SENTINEL).all())
    return out, untouched


def _run(fn, out, untouched):
    fn()
    first = out.clone()
    fn()
    assert torch.equal(first, out), "second launch differs"
    assert untouched(), "a store reached outside the out view"
    return first


VARIANTS = ["nobias", "bias", "residual", "residual_stats", "gated", "gated_stats", "ln_fold", "geglu", "geglu_ln_fold"]


@pytest.mark.parametrize("sk", [False, True], ids=["dp", "sk"])
@pytest.mark.parametrize("M", [77, 1000])
@pytest.mark.parametrize("variant", VARIANTS)
def test_linear_variants(cuda_device, storage, plan, variant, M, sk):
    """K = 640 (10 k-blocks: long enough for stream-K); N = 640 leaves a partial column tile at BN = 192 / 256."""
    ops = _ops()
    from instancediffusion_b200.packing import pack_geglu
    N, K, rpb = 640, 640, 250 if M == 1000 else 40
    a = _rand((M, K), cuda_device, 1.0, 1)
    w = _rand((N, K), cuda_device, 1.0 / math.sqrt(K), 2)
    bias = _rand((N,), cuda_device, 0.5, 3, half=False)
    res = _rand((M, N), cuda_device, 1.0, 4)
    h = a.float() @ w.float().t() + bias
    gr = torch.tensor([0.5, -1.25, 2.0, 0.0], device=cuda_device)
    gr_rows = gr.repeat_interleave(rpb)[:M, None]
    bns = [256] if variant.startswith("geglu") else ([128, 160, 192] if variant.startswith("gated") else [128, 160, 192, 256])
    for bn in bns:
        plan(bn, sk)
        out, untouched = _strided_out(M, N, cuda_device)  # (GEGLU: 2N packed columns -> N outputs)
        stats = None
        if variant == "nobias":
            fn, ref = (lambda: ops.gemm(a, w, out=out)), a.float() @ w.float().t()
        elif variant == "bias":
            fn, ref = (lambda: ops.gemm(a, w, bias, out=out)), h
        elif variant == "residual":
            fn, ref = (lambda: ops.gemm(a, w, bias, residual=res, gate=0.37, out=out)), res.float() + 0.37 * h
        elif variant == "residual_stats":
            holder = {}

            def fn():
                holder["st"] = ops.gemm(a, w, bias, residual=res, gate=0.37, out=out, want_stats=True)[1]
            ref, stats = res.float() + 0.37 * h, holder
        elif variant in ("gated", "gated_stats"):
            holder = {}

            def fn():
                r = ops.gemm(a, w, bias, residual=res, gate=0.8, gate_rows=gr, rows_per_batch=rpb, out=out,
                             want_stats=variant == "gated_stats")
                if variant == "gated_stats":
                    holder["st"] = r[1]
            ref = res.float() + 0.8 * gr_rows * h
            stats = holder if variant == "gated_stats" else None
        else:
            x, st = ops.gemm(a, w, bias, residual=res, gate=0.7, want_stats=True)
            gamma = 1.0 + 0.3 * _rand((N,), cuda_device, 1.0, 5, half=False)
            beta = 0.2 * _rand((N,), cuda_device, 1.0, 6, half=False)
            ln_ref = F.layer_norm(x.float(), (N,), gamma, beta, 1e-5)
            if variant == "ln_fold":
                w1 = _rand((N, N), cuda_device, 1.0 / math.sqrt(N), 7, half=False)
                b1 = _rand((N,), cuda_device, 0.3, 8, half=False)
                f1 = ops.fold_layernorm(w1, b1, gamma, beta, 1e-5)
                fn = lambda: ops.gemm(x, f1.w, f1.bias, ln=(st, f1.colsum, f1.eps), out=out)
                ref, tol = ln_ref @ w1.t() + b1, 4e-3
            else:
                wg = _rand((2 * N, N), cuda_device, 1.0 / math.sqrt(N), 9, half=False)
                bg = _rand((2 * N,), cuda_device, 0.3, 10, half=False)
                if variant == "geglu":
                    wp, bp = pack_geglu(wg.to(ops.HALF), bg)
                    fn = lambda: ops.gemm(x, wp, bp, geglu=True, out=out)
                    v, g = (x.float() @ wg.to(ops.HALF).float().t() + bg).chunk(2, dim=-1)
                else:
                    fg = ops.fold_layernorm(wg, bg, gamma, beta, 1e-5, pack=pack_geglu)
                    fn = lambda: ops.gemm(x, fg.w, fg.bias, geglu=True, ln=(st, fg.colsum, fg.eps), out=out)
                    v, g = (ln_ref @ wg.t() + bg).chunk(2, dim=-1)
                ref, tol = v * F.gelu(g), 4e-3
        got = _run(fn, out, untouched)
        _close(got, ref, storage, f"{variant} M={M} bn={bn} sk={sk}", **({"tol": tol} if variant.endswith(("ln_fold", "geglu")) else {}))
        if stats is not None:  # the statistics are of the fp32 results, before rounding to 16 bits
            _close(stats["st"].t[:, :, 0].sum(0), ref.float().sum(1), storage, f"{variant} stats bn={bn}", tol=2e-2)


@pytest.mark.parametrize("shape", [(3, 5, 8, 64, 96), (2, 16, 16, 64, 320), (4, 8, 8, 128, 256), (1, 6, 12, 128, 128)])
@pytest.mark.parametrize("variant", ["rowadd", "residual"])
def test_conv_variants(cuda_device, storage, variant, shape):
    """conv3x3 + per-image row-add (ResBlock conv1) and conv3x3 + residual (conv2); patches that reach past H and
    past B (B = 3, H = 5, W = 8: patch 8 x 8 x 2) clip, sentinels after the output stay."""
    ops = _ops()
    B, H, W, Cin, Cout = shape
    M = B * H * W
    x = _rand((B, H, W, Cin), cuda_device, 1.0, 1)
    wc = _rand((Cout, Cin, 3, 3), cuda_device, 1.0 / math.sqrt(9 * Cin), 2)
    w = wc.permute(0, 2, 3, 1).reshape(Cout, 9 * Cin).contiguous()
    bias = _rand((Cout,), cuda_device, 0.5, 3, half=False)
    obuf = torch.full((M + 64, Cout), SENTINEL, dtype=ops.HALF, device=cuda_device)
    out = obuf[:M]
    y = F.conv2d(x.float().permute(0, 3, 1, 2), wc.float(), bias, padding=1)
    if variant == "rowadd":
        radd = _rand((B, 2 * Cout), cuda_device, 1.0, 5)[:, :Cout]  # a column slice: ldra != N
        fn = lambda: ops.gemm(x, w, bias, conv=(B, H, W, Cin), rowadd=radd, out=out)
        ref = (y + radd.float()[:, :, None, None]).permute(0, 2, 3, 1).reshape(M, Cout)
    else:
        res = _rand((M, Cout), cuda_device, 1.0, 4)
        fn = lambda: ops.gemm(x, w, bias, conv=(B, H, W, Cin), residual=res, out=out)
        ref = y.permute(0, 2, 3, 1).reshape(M, Cout) + res.float()
    fn()
    first = out.clone()
    fn()
    assert torch.equal(first, out), "second launch differs"
    _close(out, ref, storage, f"conv {variant} {shape}")
    assert (obuf[M:] == SENTINEL).all(), "a conv store reached past the output"


def test_variants_cuda_graph(cuda_device, storage):
    """A LayerNorm-folded GEMM, a GEGLU with the fold and a gated residual GEMM with statistics captured in one
    graph: replays match the eager results bitwise."""
    ops = _ops()
    from instancediffusion_b200.packing import pack_geglu
    M, C = 1000, 320
    a = _rand((M, C), cuda_device, 1.0, 1)
    w0 = _rand((C, C), cuda_device, 1.0 / math.sqrt(C), 2)
    b0 = _rand((C,), cuda_device, 0.5, 3, half=False)
    res = _rand((M, C), cuda_device, 1.0, 4)
    gr = torch.tensor([1.0, 0.5, 0.0, 2.0], device=cuda_device)
    gamma = torch.ones(C, device=cuda_device)
    beta = torch.zeros(C, device=cuda_device)
    f1 = ops.fold_layernorm(_rand((3 * C, C), cuda_device, 1.0 / math.sqrt(C), 5, half=False), None, gamma, beta, 1e-5)
    fg = ops.fold_layernorm(_rand((8 * C, C), cuda_device, 1.0 / math.sqrt(C), 6, half=False),
                            _rand((8 * C,), cuda_device, 0.3, 7, half=False), gamma, beta, 1e-5, pack=pack_geglu)
    x = torch.empty((M, C), dtype=ops.HALF, device=cuda_device)
    o1 = torch.empty((M, 3 * C), dtype=ops.HALF, device=cuda_device)
    og = torch.empty((M, 4 * C), dtype=ops.HALF, device=cuda_device)

    def run():
        _, st = ops.gemm(a, w0, b0, residual=res, gate=0.9, gate_rows=gr, rows_per_batch=250, out=x, want_stats=True)
        ops.gemm(x, f1.w, f1.bias, ln=(st, f1.colsum, f1.eps), out=o1)
        ops.gemm(x, fg.w, fg.bias, geglu=True, ln=(st, fg.colsum, fg.eps), out=og)
    with ops.capture_workspace(cuda_device):
        run()
        eager = (x.clone(), o1.clone(), og.clone())
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=s):
                run()
        torch.cuda.current_stream().wait_stream(s)
    for _ in range(2):
        for t in (x, o1, og):
            t.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert all(torch.equal(t, e) for t, e in zip((x, o1, og), eager))
