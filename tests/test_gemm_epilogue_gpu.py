"""The GEMM epilogue staged through shared memory (residual in and result out by TMA): every epilogue mode at
every tile width, data-parallel and stream-K, against torch fp32 on the same 16-bit inputs, and a second
launch bitwise equal to the first.  The edges the tensor maps must clip: M not a multiple of 128, M < 128,
N not a multiple of the tile width, strided and offset `out` / `residual` views whose neighbouring elements
must come back untouched, conv3x3 patches that reach past the image and the batch, in-place residual, and
a CUDA-graph replay.  Runs against both storage builds of the library (bf16 tolerances scaled by 8)."""
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
    """Set IDIFF_GEMM_PLAN ("bn,sk") for the test's launches."""
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


def _twice(fn):
    """Launch twice; the second result must be bitwise equal to the first."""
    first = fn().clone()
    assert torch.equal(first, fn()), "second launch differs"
    return first


MODES = ["plain", "residual", "residual_gate", "silu", "gelu", "rowadd", "gated_rows", "geglu"]


@pytest.mark.parametrize("sk", [False, True], ids=["dp", "sk"])
@pytest.mark.parametrize("bn", [128, 160, 192, 256])
@pytest.mark.parametrize("mode", MODES)
def test_epilogue_modes(cuda_device, storage, plan, mode, bn, sk):
    """M = 1000 (8 row tiles, the last one 104 rows), N = 640 (BN = 192 and 256 leave a partial column tile),
    K = 640 (10 k-blocks: long enough for the stream-K schedule)."""
    ops = _ops()
    M, N, K, rpb = 1000, 640, 640, 250
    a = _rand((M, K), cuda_device, 1.0, 1)
    w = _rand((N, K), cuda_device, 1.0 / math.sqrt(K), 2)
    bias = _rand((N,), cuda_device, 0.5, 3, half=False)
    res = _rand((M, N), cuda_device, 1.0, 4)
    h = a.float() @ w.float().t() + bias
    plan(bn, sk)
    if mode == "plain":
        fn, ref = (lambda: ops.gemm(a, w, bias)), h
    elif mode == "residual":
        fn, ref = (lambda: ops.gemm(a, w, bias, residual=res)), res.float() + h
    elif mode == "residual_gate":
        fn, ref = (lambda: ops.gemm(a, w, bias, residual=res, gate=0.37)), res.float() + 0.37 * h
    elif mode == "silu":
        fn, ref = (lambda: ops.gemm(a, w, bias, silu=True)), F.silu(h)
    elif mode == "gelu":
        fn, ref = (lambda: ops.gemm(a, w, bias, gelu=True)), F.gelu(h)
    elif mode == "rowadd":
        radd = _rand((M // rpb, N), cuda_device, 1.0, 5)
        fn = lambda: ops.gemm(a, w, bias, rowadd=radd, rows_per_batch=rpb, residual=res)
        ref = res.float() + h + radd.float().repeat_interleave(rpb, dim=0)
    elif mode == "gated_rows":
        gr = torch.tensor([0.5, -1.25, 2.0, 0.0], device=cuda_device)
        fn = lambda: ops.gemm(a, w, bias, residual=res, gate=0.8, gate_rows=gr, rows_per_batch=rpb)
        ref = res.float() + 0.8 * gr.repeat_interleave(rpb)[:, None] * h
    else:
        from instancediffusion_b200.packing import pack_geglu
        wf, bf = _rand((2 * N, K), cuda_device, 1.0 / math.sqrt(K), 6, half=False), _rand((2 * N,), cuda_device, 0.5, 7, half=False)
        wp, bp = pack_geglu(wf.to(ops.HALF), bf)
        hg = a.float() @ wf.to(ops.HALF).float().t() + bf
        v, g = hg.chunk(2, dim=-1)
        fn, ref = (lambda: ops.gemm(a, wp, bp, geglu=True)), v * F.gelu(g)
    _close(_twice(fn), ref, storage, f"{mode} bn={bn} sk={sk}")


@pytest.mark.parametrize("sk", [False, True], ids=["dp", "sk"])
@pytest.mark.parametrize("bn", [128, 160, 192, 256])
def test_epilogue_layernorm_fold(cuda_device, storage, plan, bn, sk):
    """Producer (residual + row statistics) -> plain and GEGLU consumers through the LayerNorm fold."""
    ops = _ops()
    from instancediffusion_b200.packing import pack_geglu
    M, C = 1000, 640
    a = _rand((M, C), cuda_device, 1.0, 1)
    w0 = _rand((C, C), cuda_device, 1.0 / math.sqrt(C), 2)
    b0 = _rand((C,), cuda_device, 0.5, 3, half=False)
    res = _rand((M, C), cuda_device, 1.0, 4)
    plan(bn, sk)
    x, st = ops.gemm(a, w0, b0, residual=res, gate=0.7, want_stats=True)
    xf = x.float()
    _close(x, res.float() + 0.7 * (a.float() @ w0.float().t() + b0), storage, "ln producer")
    _close(st.t[:, :, 0].sum(0), xf.sum(1), storage, "ln producer sums", tol=2e-2)
    gamma = 1.0 + 0.3 * _rand((C,), cuda_device, 1.0, 5, half=False)
    beta = 0.2 * _rand((C,), cuda_device, 1.0, 6, half=False)
    ln_ref = F.layer_norm(xf, (C,), gamma, beta, 1e-5)
    w1 = _rand((3 * C, C), cuda_device, 1.0 / math.sqrt(C), 7, half=False)
    f1 = ops.fold_layernorm(w1, None, gamma, beta, 1e-5)
    out1 = _twice(lambda: ops.gemm(x, f1.w, f1.bias, ln=(st, f1.colsum, f1.eps)))
    _close(out1, ln_ref @ w1.t(), storage, "ln consumer plain", tol=4e-3)
    wg = _rand((4 * C, C), cuda_device, 1.0 / math.sqrt(C), 8, half=False)
    bg = _rand((4 * C,), cuda_device, 0.3, 9, half=False)
    fg = ops.fold_layernorm(wg, bg, gamma, beta, 1e-5, pack=pack_geglu)
    outg = _twice(lambda: ops.gemm(x, fg.w, fg.bias, geglu=True, ln=(st, fg.colsum, fg.eps)))
    v, g = (ln_ref @ wg.t() + bg).chunk(2, dim=-1)
    _close(outg, v * F.gelu(g), storage, "ln consumer geglu", tol=4e-3)


@pytest.mark.parametrize("M", [77, 100, 300])
@pytest.mark.parametrize("bn", [128, 160, 192, 256])
def test_epilogue_strided_views(cuda_device, storage, plan, M, bn):
    """`out` and `residual` as column slices of wider buffers (ldo, ldr > N), `out` at a row offset: the
    sentinels around them (columns past N, rows before and past the view) must come back untouched."""
    ops = _ops()
    N, K = 320, 320
    a = _rand((M, K), cuda_device, 1.0, 1)
    w = _rand((N, K), cuda_device, 1.0 / math.sqrt(K), 2)
    bias = _rand((N,), cuda_device, 0.5, 3, half=False)
    rbuf = _rand((M + 9, N + 40), cuda_device, 1.0, 4)
    res = rbuf[5:5 + M, 8:8 + N]
    obuf = torch.full((M + 13, N + 72), SENTINEL, dtype=ops.HALF, device=cuda_device)
    out = obuf[3:3 + M, 16:16 + N]
    plan(bn, False)
    _twice(lambda: ops.gemm(a, w, bias, residual=res, gate=0.5, out=out))
    _close(out, res.float() + 0.5 * (a.float() @ w.float().t() + bias), storage, f"strided M={M} bn={bn}")
    mask = torch.ones_like(obuf, dtype=torch.bool)
    mask[3:3 + M, 16:16 + N] = False
    assert (obuf[mask] == SENTINEL).all(), "a store reached outside the out view"


@pytest.mark.parametrize("bn", [128, 160, 192, 256])
def test_epilogue_in_place_residual(cuda_device, storage, plan, bn):
    """residual is out (the transformer blocks' proj_out / attention outputs): bitwise equal to out-of-place."""
    ops = _ops()
    M, N, K = 1000, 640, 320
    a = _rand((M, K), cuda_device, 1.0, 1)
    w = _rand((N, K), cuda_device, 1.0 / math.sqrt(K), 2)
    bias = _rand((N,), cuda_device, 0.5, 3, half=False)
    x = _rand((M, N), cuda_device, 1.0, 4)
    plan(bn, False)
    ref = ops.gemm(a, w, bias, residual=x, gate=0.9)
    ops.gemm(a, w, bias, residual=x, gate=0.9, out=x)
    assert torch.equal(x, ref)


@pytest.mark.parametrize("shape", [(3, 5, 8, 64, 96), (2, 16, 16, 64, 320), (1, 6, 12, 128, 128)])
def test_epilogue_conv3x3(cuda_device, storage, shape):
    """Implicit-GEMM conv3x3 with residual and per-image row-add; patches that reach past H and past B
    (B=3, H=5, W=8: patch 8 x 8 x 2) must not write outside the output, whose trailing rows hold sentinels."""
    ops = _ops()
    B, H, W, Cin, Cout = shape
    M = B * H * W
    x = _rand((B, H, W, Cin), cuda_device, 1.0, 1)
    wc = _rand((Cout, Cin, 3, 3), cuda_device, 1.0 / math.sqrt(9 * Cin), 2)
    w = wc.permute(0, 2, 3, 1).reshape(Cout, 9 * Cin).contiguous()  # K index = (ky * 3 + kx) * Cin + ci
    bias = _rand((Cout,), cuda_device, 0.5, 3, half=False)
    res = _rand((M, Cout), cuda_device, 1.0, 4)
    radd = _rand((B, Cout), cuda_device, 1.0, 5)
    obuf = torch.full((M + 64, Cout), SENTINEL, dtype=ops.HALF, device=cuda_device)
    out = obuf[:M]
    _twice(lambda: ops.gemm(x, w, bias, conv=(B, H, W, Cin), residual=res, rowadd=radd, out=out))
    y = F.conv2d(x.float().permute(0, 3, 1, 2), wc.float(), bias, padding=1) + radd.float()[:, :, None, None]
    ref = y.permute(0, 2, 3, 1).reshape(M, Cout) + res.float()
    _close(out, ref, storage, f"conv3x3 {shape}")
    assert (obuf[M:] == SENTINEL).all(), "a conv store reached past the output"


def test_epilogue_cuda_graph(cuda_device, storage):
    """Capture a residual GEMM and a stream-K one into a graph; replays match the eager results bitwise."""
    ops = _ops()
    a = _rand((1000, 640), cuda_device, 1.0, 1)
    w = _rand((640, 640), cuda_device, 1.0 / math.sqrt(640), 2)
    bias = _rand((640,), cuda_device, 0.5, 3, half=False)
    res = _rand((1000, 640), cuda_device, 1.0, 4)
    a2 = _rand((2048, 5120), cuda_device, 1.0, 5)
    w2 = _rand((1280, 5120), cuda_device, 1.0 / math.sqrt(5120), 6)
    b2 = _rand((1280,), cuda_device, 0.5, 7, half=False)
    out = torch.empty((1000, 640), dtype=ops.HALF, device=cuda_device)
    out2 = torch.empty((2048, 1280), dtype=ops.HALF, device=cuda_device)
    run = lambda: (ops.gemm(a, w, bias, residual=res, out=out), ops.gemm(a2, w2, b2, residual=out2, out=out2))
    with ops.capture_workspace(cuda_device):
        out2.zero_()
        run()
        eager = (out.clone(), out2.clone())
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=s):
                run()
        torch.cuda.current_stream().wait_stream(s)
    for _ in range(2):
        out.zero_()
        out2.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, eager[0]) and torch.equal(out2, eager[1])
