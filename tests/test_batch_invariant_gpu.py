"""`-m gpu` tests of batch-invariant mode (ops.set_batch_invariant): with the mode on, an image computed alone and the
same image inside batches of 2, 3, 8, 17 and 32 with different random neighbours, at different positions, give the
same bits -- for the kernels (every GEMM epilogue, conv3x3, GroupNorm, ScaleU, attention), for
UNetModel.forward_batched, and for the request drivers against each request's own sampler run."""
import os
import sys
from functools import partial

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from test_engine_gpu import _drive, _requests  # noqa: E402
from test_requests_gpu import _att_masks, _fresh, _reset, _run_alone  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(HERE, "golden")
BATCHES = (2, 3, 8, 17, 32)
DTYPES = [torch.float16, torch.bfloat16]


@pytest.fixture(params=DTYPES, ids=["fp16", "bf16"])
def storage(request, cuda_device):
    """The model and driver cases in both storage types."""
    from instancediffusion_b200 import ops
    with ops.storage(request.param):
        yield request.param


@pytest.fixture
def invariant(cuda_device):
    from instancediffusion_b200 import ops
    ops.set_batch_invariant(True)
    yield
    ops.set_batch_invariant(False)


def _batches(make, n_max=32, batches=BATCHES, seed=0):
    """(image 0 alone, [(position, batch of n images with image 0 at position)]) from make(n) -> n per-image items."""
    pool = make(n_max)
    g = torch.Generator().manual_seed(seed)
    out = []
    for n in batches:
        others = [1 + int(i) for i in torch.randperm(n_max - 1, generator=g)[:n - 1]]
        pos = (n * 5 // 7) % n
        order = others[:pos] + [0] + others[pos:]
        out.append((pos, [pool[i] for i in order]))
    return pool[0], out


def _check_rows(run, per_image, batches, what):
    """run(list of per-image items) -> tensor whose leading dimension is grouped by image (or a tuple of them): image
    0's slice of every batch equals its result alone, bit for bit."""
    alone = run([per_image])
    alone = alone if isinstance(alone, tuple) else (alone,)
    for pos, items in batches:
        got = run(items)
        got = got if isinstance(got, tuple) else (got,)
        for k, (a, b) in enumerate(zip(alone, got)):
            n = a.shape[0]
            assert torch.equal(b[pos * n:(pos + 1) * n], a), \
                f"{what}: output {k} of image 0 at position {pos} of {len(items)} differs"


# ------------------------------------------------------------------------------------------------
# 1. GEMM epilogues, conv3x3, the stride-2 operand
# ------------------------------------------------------------------------------------------------
def _rand(g, shape, scale=1.0):
    return torch.randn(shape, generator=g) * scale


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("epi", ["bias", "residual", "silu_rowadd", "gelu", "geglu", "gate_rows", "ln_fold"])
@pytest.mark.parametrize("R,N,K", [(77, 640, 640), (256, 1280, 1280), (300, 320, 768)])
def test_gemm_epilogues(cuda_device, invariant, dtype, epi, R, N, K):
    from instancediffusion_b200 import ops
    g = torch.Generator().manual_seed(R + N + K)
    dev = cuda_device
    with ops.storage(dtype):
        w = (_rand(g, (N * (2 if epi == "geglu" else 1), K)) / K ** 0.5).to(dev, dtype)
        bias = _rand(g, (w.shape[0],), 0.1).to(dev)
        colsum = w.float().sum(1).contiguous()
        wsq = (_rand(g, (K, K)) / K ** 0.5).to(dev, dtype)

        def make(n):
            return [dict(a=_rand(g, (R, K), 0.5).to(dev, dtype), res=_rand(g, (R, N)).to(dev, dtype),
                         add=_rand(g, (1, N), 0.3).to(dev, dtype), gate=float(_rand(g, (1,))))
                    for _ in range(n)]

        def run(items):
            a = torch.cat([i["a"] for i in items])
            res = torch.cat([i["res"] for i in items])
            if epi == "bias":
                return ops.gemm(a, w, bias)
            if epi == "residual":
                out, st = ops.gemm(a, w, bias, residual=res, gate=0.7, want_stats=True)
                return out, st.t.transpose(0, 1).contiguous()
            if epi == "silu_rowadd":
                return ops.gemm(a, w, bias, rowadd=torch.cat([i["add"] for i in items]), rows_per_batch=R, silu=True)
            if epi == "gelu":
                return ops.gemm(a, w, bias, gelu=True)
            if epi == "geglu":
                return ops.gemm(a, w, bias, geglu=True) if N % 128 == 0 else ops.gemm(a, w, bias)
            rows = torch.tensor([i["gate"] for i in items], dtype=torch.float32, device=dev)
            if epi == "gate_rows":
                out, st = ops.gemm(a, w, bias, residual=res, gate=0.6, gate_rows=rows, rows_per_batch=R, want_stats=True)
                return out, st.t.transpose(0, 1).contiguous()
            # LayerNorm fold out of one GEMM (producer statistics) and into the next
            h, st = ops.gemm(a, wsq, None, residual=a, want_stats=True)
            y = ops.gemm(h, w, bias, ln=(st, colsum, 1e-5))
            return h, y, st.t.transpose(0, 1).contiguous()

        one, bs = _batches(make)
        _check_rows(run, one, bs, f"gemm {epi} R={R} N={N} K={K}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("S,cin,cout", [(64, 320, 320), (32, 640, 640), (16, 1280, 1280), (8, 1280, 1280),
                                        (12, 640, 1280), (64, 320, 4)])
def test_conv3x3(cuda_device, invariant, dtype, S, cin, cout):
    from instancediffusion_b200 import ops
    from instancediffusion_b200.packing import pack_conv3x3
    g = torch.Generator().manual_seed(S * cin + cout)
    dev = cuda_device
    with ops.storage(dtype):
        w = pack_conv3x3((_rand(g, (cout, cin, 3, 3)) / (9 * cin) ** 0.5).to(dev, dtype))
        bias = _rand(g, (cout,), 0.1).to(dev)

        def make(n):
            return [dict(x=_rand(g, (S * S, cin)).to(dev, dtype), res=_rand(g, (S * S, cout)).to(dev, dtype),
                         add=_rand(g, (1, cout), 0.3).to(dev, dtype)) for _ in range(n)]

        def run(items):
            B = len(items)
            x = torch.cat([i["x"] for i in items])
            if cout == 4:  # the final conv: fp32 NCHW output
                eps = torch.empty((B, 4, S, S), dtype=torch.float32, device=dev)
                ops.gemm(x, w, bias, conv=(B, S, S, cin), out_nchw=eps)
                return eps
            y = ops.gemm(x, w, bias, conv=(B, S, S, cin), rowadd=torch.cat([i["add"] for i in items]))
            z = ops.gemm(x, w, bias, conv=(B, S, S, cin), residual=torch.cat([i["res"] for i in items]))
            return y, z

        one, bs = _batches(make, batches=BATCHES if S <= 32 or cin <= 320 else (2, 3, 8))
        _check_rows(run, one, bs, f"conv3x3 {S}x{S} {cin}->{cout}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("S,c", [(64, 320), (32, 640), (16, 1280)])
def test_downsample_operand(cuda_device, invariant, dtype, S, c):
    from instancediffusion_b200 import ops
    from instancediffusion_b200.packing import pack_conv3x3
    g = torch.Generator().manual_seed(S + c)
    dev = cuda_device
    with ops.storage(dtype):
        w = pack_conv3x3((_rand(g, (c, c, 3, 3)) / (9 * c) ** 0.5).to(dev, dtype))
        bias = _rand(g, (c,), 0.1).to(dev)
        one, bs = _batches(lambda n: [_rand(g, (S * S, c)).to(dev, dtype) for _ in range(n)], batches=(2, 3, 8, 17))
        _check_rows(lambda items: ops.gemm(ops.im2col_s2(torch.cat(items), len(items), S, S), w, bias), one, bs,
                    f"downsample {S}x{S} {c}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("C,R", [(320, 4096), (640, 1024), (1280, 256), (1280, 64)])
def test_gate_zero_keeps_producer_statistics(cuda_device, invariant, dtype, C, R):
    """What makes a skipped fuser and a fuser gated to 0 agree: a per-image-gated GEMM passes a gate-0 image's residual
    rows through unchanged and writes the LayerNorm statistics the plain GEMM that produced them wrote, over the same
    slots."""
    from instancediffusion_b200 import ops
    g = torch.Generator().manual_seed(C + R)
    dev = cuda_device
    B = 3
    with ops.storage(dtype):
        x = _rand(g, (B * R, C)).to(dev, dtype)
        a, a2 = (_rand(g, (B * R, C), 0.5).to(dev, dtype) for _ in range(2))
        w, w2 = ((_rand(g, (C, C)) / C ** 0.5).to(dev, dtype) for _ in range(2))
        bias, bias2 = (_rand(g, (C,), 0.1).to(dev) for _ in range(2))
        h, st = ops.gemm(a, w, bias, residual=x, want_stats=True)  # (the attention out-projection before the fuser)
        rows = torch.tensor([0.0, 0.7, 0.0], dtype=torch.float32, device=dev)
        out, st2 = ops.gemm(a2, w2, bias2, residual=h, gate=0.9, gate_rows=rows, rows_per_batch=R, want_stats=True)
        assert st2.slots == st.slots
        for b in (0, 2):
            r = slice(b * R, (b + 1) * R)
            assert torch.equal(out[r], h[r]), b
            assert torch.equal(st2.t[:, r], st.t[:, r]), b


def test_gemm_plan_override_keeps_data_parallel(cuda_device, invariant, monkeypatch):
    """IDIFF_GEMM_PLAN (a tuning knob that can force stream-K) has no effect in the mode."""
    from instancediffusion_b200 import ops
    g = torch.Generator().manual_seed(5)
    a = _rand(g, (17 * 300, 1280), 0.5).to(cuda_device, ops.HALF)
    w = (_rand(g, (1280, 1280)) / 1280 ** 0.5).to(cuda_device, ops.HALF)
    ref = ops.gemm(a, w)
    monkeypatch.setenv("IDIFF_GEMM_PLAN", "128,1")
    assert torch.equal(ops.gemm(a, w), ref)
    assert torch.equal(ops.gemm(a[:300], w), ref[:300])


# ------------------------------------------------------------------------------------------------
# 2. GroupNorm, ScaleU, attention
# ------------------------------------------------------------------------------------------------
GN_SHAPES = [  # (hw side, C, eps, silu): UNet ResBlocks / SpatialTransformers / out, VAE decoder
    (64, 320, 1e-5, True), (64, 640, 1e-5, True), (64, 960, 1e-5, True), (32, 320, 1e-5, True), (32, 640, 1e-5, True),
    (32, 960, 1e-5, True), (32, 1280, 1e-5, True), (32, 1920, 1e-5, True), (16, 640, 1e-5, True),
    (16, 1280, 1e-5, True), (16, 1920, 1e-5, True), (16, 2560, 1e-5, True), (8, 1280, 1e-5, True),
    (8, 2560, 1e-5, True), (64, 320, 1e-6, False), (32, 640, 1e-6, False), (16, 1280, 1e-6, False),
    (8, 1280, 1e-6, False), (64, 512, 1e-6, True), (128, 512, 1e-6, True), (256, 512, 1e-6, True),
    (256, 256, 1e-6, True), (512, 256, 1e-6, True), (512, 128, 1e-6, True), (64, 512, 1e-6, False),
]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("S,C,eps,silu", GN_SHAPES)
def test_groupnorm(cuda_device, invariant, dtype, S, C, eps, silu):
    from instancediffusion_b200 import ops
    g = torch.Generator().manual_seed(S * C)
    dev = cuda_device
    gamma = (1 + _rand(g, (C,), 0.1)).to(dev)
    beta = _rand(g, (C,), 0.1).to(dev)
    per_image = S * S * C
    n_max = max(3, min(32, (1 << 27) // per_image))
    batches = tuple(b for b in BATCHES if b <= n_max)
    with ops.storage(dtype):
        one, bs = _batches(lambda n: [(_rand(g, (S * S, C)) * 2 + 0.5).to(dev, dtype) for _ in range(n)],
                           n_max=n_max, batches=batches)
        _check_rows(lambda items: ops.groupnorm(torch.cat(items), gamma, beta, batch=len(items), hw=S * S, groups=32,
                                                eps=eps, silu=silu), one, bs, f"groupnorm {S}x{S} C={C}")


SCALEU_SITES = [(8, 1280, 1280)] * 3 + [(16, 1280, 1280), (16, 1280, 1280), (16, 1280, 640), (32, 1280, 640),
                                        (32, 640, 640), (32, 640, 320), (64, 640, 320), (64, 320, 320), (64, 320, 320)]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("site", range(12))
def test_scaleu_concat(cuda_device, invariant, dtype, site):
    from instancediffusion_b200 import ops
    S, c1, c2 = SCALEU_SITES[site]
    g = torch.Generator().manual_seed(site)
    dev = cuda_device
    b1 = (1 + _rand(g, (c1,), 0.2)).to(dev)
    with ops.storage(dtype):
        def make(n):
            return [(_rand(g, (S * S, c1)).to(dev, dtype), _rand(g, (S * S, c2)).to(dev, dtype)) for _ in range(n)]
        one, bs = _batches(make)
        _check_rows(lambda items: ops.scaleu_concat(torch.cat([h for h, _ in items]), torch.cat([s for _, s in items]),
                                                    b1, 1.3, batch=len(items), height=S, width=S),
                    one, bs, f"scaleu site {site}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("d,segment,mask", [(40, False, False), (40, True, False), (40, True, True), (80, False, False),
                                            (80, True, False), (160, False, False), (160, True, False)])
def test_attention(cuda_device, invariant, dtype, d, segment, mask):
    from instancediffusion_b200 import ops
    heads, nq = 8, {40: 4096, 80: 1024, 160: 256}[d]
    n_obj = 184
    C = heads * d
    g = torch.Generator().manual_seed(d + 2 * segment + mask)
    dev = cuda_device
    with ops.storage(dtype):
        def make(n):
            out = []
            for _ in range(n):
                it = dict(qkv=_rand(g, (nq, 3 * C)).to(dev, dtype), kv1=_rand(g, (n_obj, 2 * C)).to(dev, dtype))
                if mask:
                    boxes = torch.rand((1, 30, 4), generator=g)
                    boxes = torch.cat([boxes[..., :2] * 0.5, boxes[..., :2] * 0.5 + 0.2 + boxes[..., 2:] * 0.3], -1)
                    att = ops.boxes_to_attmask(boxes.to(dev), torch.tensor([5], dtype=torch.int32, device=dev))
                    it["mask"] = ops.attmask_words(att, torch.ones(1, dtype=torch.int32, device=dev), tail=n_obj - 4 * 30)
                out.append(it)
            return out

        def run(items):
            B = len(items)
            qkv = torch.cat([i["qkv"] for i in items])
            kw = {}
            if segment:
                kv1 = torch.cat([i["kv1"] for i in items])
                kw = dict(k1=kv1[:, :C], v1=kv1[:, C:], n1=n_obj)
            if mask:
                kw["mask"] = (torch.cat([i["mask"][0] for i in items]), torch.cat([i["mask"][1] for i in items]))
            return ops.attention(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], batch=B, heads=heads, head_dim=d, nq=nq,
                                 n0=nq, scale=d ** -0.5, **kw)

        one, bs = _batches(make, batches=BATCHES if d > 40 else (2, 3, 8, 17))
        _check_rows(run, one, bs, f"attention d={d}")


# ------------------------------------------------------------------------------------------------
# 3. UNetModel.forward_batched
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def unet(cuda_device):
    from instancediffusion_b200.weights import build_unet
    model = build_unet("box", cuda_device, seed=0)
    model._sd_conv = torch.load(os.path.join(GOLDEN, "sd15_first_conv.pt"), map_location="cpu")
    model.restore_first_conv_from_SD = lambda: (None if getattr(model, "_first_conv_restored", False)
                                                else model.set_sd_first_conv(model._sd_conv))
    model.restore_first_conv_from_SD()  # the SD1.5 weights are known from here on
    model.undo_first_conv_restore()
    yield model
    model.use_cuda_graph = True


@pytest.fixture(scope="module")
def diffusion(cuda_device):
    from instancediffusion_b200.ldm.models.diffusion.ldm import LatentDiffusion
    return LatentDiffusion(linear_start=0.00085, linear_end=0.012, timesteps=1000).to(cuda_device)


@pytest.mark.parametrize("size", [64, 96])
@pytest.mark.parametrize("graph", [False, True])
def test_forward_batched(cuda_device, unet, storage, invariant, size, graph):
    from instancediffusion_b200 import synthetic
    from instancediffusion_b200.utils.model import set_alpha_scale
    gti = unet.grounding_tokenizer_input
    inputs, scales, restored = [], [], []
    for k, seed in enumerate(range(301, 306)):
        ia, uca = synthetic.make_sampler_inputs(gti, 1, 2, seed, "box", device=cuda_device, size=size)
        if size == 64 and k == 1:
            ia["grounding_input"]["att_masks"] = _att_masks(ia["grounding_input"])
        t = torch.full((1,), 100 + 150 * k, dtype=torch.long, device=cuda_device)
        inputs += [dict(x=ia["x"], timesteps=t, context=ia["context"], grounding_input=ia["grounding_input"]),
                   dict(x=ia["x"] * 0.7, timesteps=t, context=uca)]
        scales += [(1.0, 0.0, 0.36, 1.0, 0.0)[k]] * 2
        restored += [k % 2 == 1] * 2
    unet.use_cuda_graph = graph
    try:
        _reset(unet)
        refs = []
        for inp, s, r in zip(inputs, scales, restored):  # each input alone, as its own sample() runs it
            set_alpha_scale(unet, s)
            if r:
                unet.restore_first_conv_from_SD()
            refs.append(unet(dict(inp)).clone())
            unet.undo_first_conv_restore()
        set_alpha_scale(unet, 1)
        for perm in (list(range(len(inputs))), list(reversed(range(len(inputs)))), [3, 0, 7, 2]):
            ins = [inputs[i] for i in perm]
            for kw in (dict(per_image_conv=True), dict()):
                got = unet.forward_batched(ins, scales=[scales[i] for i in perm], restored=[restored[i] for i in perm], **kw)
                for j, i in enumerate(perm):
                    assert torch.equal(got[j], refs[i]), (perm, kw, i)
    finally:
        _reset(unet)
        unet.use_cuda_graph = True


def test_mode_switch_drops_graphs(cuda_device, unet, storage):
    """A graph captured in one mode is never replayed in the other: the model drops its graphs and hoisted tensors on
    the switch, and each mode's result equals that mode's eager result."""
    from instancediffusion_b200 import ops, synthetic
    gti = unet.grounding_tokenizer_input
    ia, uca = synthetic.make_sampler_inputs(gti, 1, 2, 311, "box", device=cuda_device)
    t = torch.full((1,), 500, dtype=torch.long, device=cuda_device)
    inputs = [dict(x=ia["x"], timesteps=t, context=ia["context"], grounding_input=ia["grounding_input"]),
              dict(x=ia["x"], timesteps=t, context=uca)]
    _reset(unet)
    try:
        eager = {}
        unet.use_cuda_graph = False
        for mode in (False, True):
            ops.set_batch_invariant(mode)
            eager[mode] = unet.forward_batched(inputs, scales=[1.0, 0.36])
        unet.use_cuda_graph = True
        seen = {}
        for mode in (False, True, False, True):
            ops.set_batch_invariant(mode)
            got = unet.forward_batched(inputs, scales=[1.0, 0.36])
            graphs = list(unet._graphs.values())  # (the objects themselves: a dropped graph's id may be reused)
            assert not any(g is h for g in graphs for h in seen.get(not mode, [])), \
                "a graph of the other mode survived the switch"
            seen[mode] = graphs
            for a, b in zip(got, eager[mode]):
                assert torch.equal(a, b), mode
        assert not all(torch.equal(a, b) for a, b in zip(eager[True], eager[False]))
    finally:
        ops.set_batch_invariant(False)
        _reset(unet)


# ------------------------------------------------------------------------------------------------
# 4. drivers
# ------------------------------------------------------------------------------------------------
def _driver_requests(unet, device, S):
    """Plain, MIS 0.36 (n = 3, one with the instance-isolation mask), MIS 1.0 and no alpha schedule, at S steps."""
    from instancediffusion_b200 import synthetic
    from instancediffusion_b200.ldm.models.diffusion.batched import Request
    from instancediffusion_b200.utils.model import alpha_generator
    gti = unet.grounding_tokenizer_input
    agen = partial(alpha_generator, type=[0.8, 0.0, 0.2])
    out = []
    for seed, n, mis, alpha in ((401, 2, 0.0, agen), (402, 3, 0.36, agen), (403, 2, 1.0, agen), (404, 3, 0.0, None),
                                (405, 3, 0.36, partial(alpha_generator, type=[0.5, 0.0, 0.5]))):
        inputs, uc = synthetic.make_sampler_inputs(gti, 1, n, seed, "box", mis=mis > 0, device=device)
        if seed == 402:
            for inp in inputs:
                inp["grounding_input"]["att_masks"] = _att_masks(inp["grounding_input"])
        out.append(Request(input=inputs, uc=uc, guidance_scale=7.5, alpha_generator_func=alpha, mis=mis,
                           shape=(1, 4, 64, 64), S=S))
    return out


@pytest.mark.parametrize("S", [10, 11])
def test_sample_requests_equal_own_sample(cuda_device, unet, diffusion, storage, invariant, S):
    from instancediffusion_b200.ldm.models.diffusion.batched import sample_requests
    reqs = _driver_requests(unet, cuda_device, S)
    alone = [_run_alone(unet, diffusion, r, S) for r in reqs]
    for max_batch in (8, 32):
        _reset(unet)
        got = sample_requests(unet, diffusion, [_fresh(r) for r in reqs], S, max_batch=max_batch)
        _reset(unet)
        for j, a in enumerate(alone):
            assert torch.equal(got[j], a), (max_batch, j)


@pytest.mark.parametrize("graph", [False, True])
def test_engine_equal_own_sample(cuda_device, unet, diffusion, storage, invariant, graph):
    from instancediffusion_b200.ldm.models.diffusion.engine import SamplingEngine
    from dataclasses import replace
    reqs = _driver_requests(unet, cuda_device, 10)
    reqs[1], reqs[3] = replace(reqs[1], S=11), replace(reqs[3], S=11)
    reqs += _requests(unet, cuda_device)[2:3]  # S = 20, MIS 1.0, arriving late
    alone = [_run_alone(unet, diffusion, r, r.S) for r in reqs]
    unet.use_cuda_graph = graph
    try:
        for buckets in ((2, 4, 8), None):
            _reset(unet)
            got = _drive(SamplingEngine(unet, diffusion, max_batch=8, buckets=buckets), reqs, [0, 0, 2, 3, 5, 9])
            for j, a in enumerate(alone):
                assert torch.equal(got[j], a), (buckets, j)
    finally:
        _reset(unet)
        unet.use_cuda_graph = True
