"""`-m gpu` tests of batched request sampling: the per-image residual gate of the GEMM epilogue (idiff_gemm_args.gate_b),
UNetModel.forward_batched(scales=, restored=) against separate forwards, and sample_requests against each request's own
sampler run -- plus one request anchored to the reference's golden latent."""
import os
import sys
from functools import partial

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import cases  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(HERE, "golden")
EPS_TOL = 4e-3        # as test_parity_r2_gpu.py
LATENT_TOL = 4.4e-3
S_TEST = 10


def _rel(got, ref):
    got, ref = got.detach().float().cpu(), ref.detach().float().cpu()
    assert got.shape == ref.shape, (tuple(got.shape), tuple(ref.shape))
    assert torch.isfinite(got).all()
    return ((got - ref).norm() / ref.norm()).item()


# ------------------------------------------------------------------------------------------------
# 1. kernel: gate_b in the gated-residual epilogue
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("M,rpb,N,K", [(2 * 4096, 4096, 320, 320), (3 * 1024, 1024, 640, 640), (5 * 64, 64, 1280, 1280),
                                       (4 * 256, 256, 640, 2560)])
def test_gemm_gate_rows(cuda_device, monkeypatch, dtype, M, rpb, N, K):
    from instancediffusion_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(M + N)
    B = M // rpb
    with ops.storage(dtype):
        a = (torch.randn((M, K), generator=g) * 0.5).to(cuda_device, dtype)
        w = (torch.randn((N, K), generator=g) / K ** 0.5).to(cuda_device, dtype)
        bias = (torch.randn((N,), generator=g) * 0.1).to(cuda_device)
        res = torch.randn((M, N), generator=g).to(cuda_device, dtype)
        gate = 0.7
        rows = torch.tensor(([1.0, 0.0, -0.5, 2.0, 0.25] * 2)[:B], dtype=torch.float32, device=cuda_device)
        out = ops.gemm(a, w, bias, residual=res, gate=gate, gate_rows=rows, rows_per_batch=rpb)
        ref = res.float() + gate * rows.repeat_interleave(rpb)[:, None] * (a.float() @ w.float().t() + bias)
        r = _rel(out, ref)
        assert r < (2e-3 if dtype == torch.float16 else 1.2e-2), r
        # a zero factor leaves the residual row untouched, bit for bit
        zero = (rows == 0).repeat_interleave(rpb)
        assert torch.equal(out[zero], res[zero])
        # the scalar path (gate_rows=None) is the same result as unit factors, bit for bit, on the same tile plan
        # (gated GEMMs never take 256-wide tiles)
        monkeypatch.setenv("IDIFF_GEMM_PLAN", "160,0")
        plain = ops.gemm(a, w, bias, residual=res, gate=gate)
        ones = ops.gemm(a, w, bias, residual=res, gate=gate, gate_rows=torch.ones_like(rows), rows_per_batch=rpb)
        monkeypatch.delenv("IDIFF_GEMM_PLAN")
        assert torch.equal(plain, ones)
        # the row statistics of the folded LayerNorm are those of the stored rows
        o2, st = ops.gemm(a, w, bias, residual=res, gate=gate, gate_rows=rows, rows_per_batch=rpb, want_stats=True)
        assert torch.equal(o2, out)
        s = st.t.sum(0)  # (sums of the fp32 values before rounding to the storage type)
        stored = out.float()
        assert ((s[:, 0] - stored.sum(1)).abs() <= 8e-3 * stored.abs().sum(1) + 1e-3).all()


def test_gemm_gate_rows_needs_residual(cuda_device):
    from instancediffusion_b200 import ops
    from instancediffusion_b200._lib import IdiffError
    a = torch.zeros((128, 64), dtype=ops.HALF, device=cuda_device)
    w = torch.zeros((64, 64), dtype=ops.HALF, device=cuda_device)
    with pytest.raises(IdiffError):
        ops.gemm(a, w, gate_rows=torch.ones(1, device=cuda_device))


# ------------------------------------------------------------------------------------------------
# model fixtures
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def unet(cuda_device):
    from instancediffusion_b200.weights import build_unet
    model = build_unet("box", cuda_device, seed=0)
    model._sd_conv = torch.load(os.path.join(GOLDEN, "sd15_first_conv.pt"), map_location="cpu")
    model.restore_first_conv_from_SD = lambda: (None if getattr(model, "_first_conv_restored", False)
                                                else model.set_sd_first_conv(model._sd_conv))
    yield model
    model.use_cuda_graph = True


@pytest.fixture(scope="module")
def diffusion(cuda_device):
    from instancediffusion_b200.ldm.models.diffusion.ldm import LatentDiffusion
    return LatentDiffusion(linear_start=0.00085, linear_end=0.012, timesteps=1000).to(cuda_device)


def _reset(unet):
    from instancediffusion_b200.utils.model import set_alpha_scale
    unet.undo_first_conv_restore()
    set_alpha_scale(unet, 1)


# ------------------------------------------------------------------------------------------------
# 2. forward_batched(scales=, restored=)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("graph", [False, True])
def test_forward_batched_per_input_scale_and_first_conv(cuda_device, unet, graph):
    from instancediffusion_b200 import synthetic
    from instancediffusion_b200.utils.model import set_alpha_scale
    gti = unet.grounding_tokenizer_input
    ia, uca = synthetic.make_sampler_inputs(gti, 1, 2, 71, "box", device=cuda_device)
    ib, _ = synthetic.make_sampler_inputs(gti, 1, 3, 72, "box", device=cuda_device)
    ts = [torch.full((1,), t, dtype=torch.long, device=cuda_device) for t in (601, 801, 401, 201)]
    inputs = [dict(x=ia["x"], timesteps=ts[0], context=ia["context"], grounding_input=ia["grounding_input"]),
              dict(x=ia["x"], timesteps=ts[1], context=uca),
              dict(x=ib["x"], timesteps=ts[2], context=ib["context"], grounding_input=ib["grounding_input"]),
              dict(x=ib["x"] * 0.5, timesteps=ts[3], context=ib["context"], grounding_input=ib["grounding_input"])]
    scales, restored = [1.0, 0.0, 0.5, 1.0], [False, True, False, True]
    unet.use_cuda_graph = graph
    try:
        _reset(unet)
        refs = []
        for inp, s, r in zip(inputs, scales, restored):
            set_alpha_scale(unet, s)
            if r:
                unet.restore_first_conv_from_SD()
            refs.append(unet(dict(inp)).clone())
            unet.undo_first_conv_restore()
        set_alpha_scale(unet, 1)
        for flags in (restored, [not r for r in restored]):  # a new flag pattern replays the same graph
            n = len(unet._graphs)
            got = unet.forward_batched(inputs, scales=scales, restored=flags)
            assert not unet._first_conv_restored, "forward_batched(restored=...) must not swap the model's conv"
            if flags is restored:
                for k, (g, ref) in enumerate(zip(got, refs)):
                    r = _rel(g, ref)
                    print(f"[forward_batched graph={graph}] input {k} scale {scales[k]} restored {restored[k]}: "
                          f"rel_l2 {r:.2e}")
                    assert r < EPS_TOL, (k, r)
            else:
                assert len(unet._graphs) == n
        # equal scales take the scalar path: the fusers' own scale does not matter
        set_alpha_scale(unet, 0)
        same = unet.forward_batched(inputs[:1] + inputs[2:3], scales=[1.0, 1.0])
        assert _rel(same[0], refs[0]) < EPS_TOL
    finally:
        _reset(unet)
        unet.use_cuda_graph = True


def test_sd_conv_given_after_capture_reaches_the_graph(cuda_device, monkeypatch):
    """A graph captured before the SD1.5 conv weights are known is replayed after set_sd_first_conv gives them, and
    again after it gives different ones: each replay runs the weights given last, as the eager forward does, and the
    model's own conv for the other images."""
    from instancediffusion_b200 import synthetic
    from instancediffusion_b200.weights import build_unet
    monkeypatch.delenv("IDIFF_PRETRAINED_DIR", raising=False)
    model = build_unet("box", cuda_device, seed=0)
    ia, uca = synthetic.make_sampler_inputs(model.grounding_tokenizer_input, 1, 2, 73, "box", device=cuda_device)
    t = torch.full((1,), 501, dtype=torch.long, device=cuda_device)
    inputs = [dict(x=ia["x"], timesteps=t, context=ia["context"], grounding_input=ia["grounding_input"]),
              dict(x=ia["x"] * 0.5, timesteps=t, context=uca)]
    scales, restored = [1.0, 0.5], [True, False]

    def both():
        model.use_cuda_graph = False
        eager = model.forward_batched(inputs, scales=scales, restored=restored)
        model.use_cuda_graph = True
        return eager, model.forward_batched(inputs, scales=scales, restored=restored)

    before = model.forward_batched(inputs, scales=scales)  # captured while no SD1.5 weights are known
    n = len(model._graphs)
    with pytest.raises(FileNotFoundError):
        model.forward_batched(inputs, scales=scales, restored=restored)
    sd_a = torch.load(os.path.join(GOLDEN, "sd15_first_conv.pt"), map_location="cpu")
    g = torch.Generator().manual_seed(7)
    sd_b = {k: v + 0.05 * torch.randn(v.shape, generator=g) for k, v in sd_a.items()}
    got = []
    for sd in (sd_a, sd_b):
        model.set_sd_first_conv(sd)  # (the second call while the first SD1.5 conv is swapped in)
        eager, graphed = both()
        assert len(model._graphs) == n
        for e, r in zip(eager, graphed):
            assert torch.equal(e, r)
        assert torch.equal(graphed[1], before[1])  # the model's own conv
        got.append(graphed)
    assert not torch.equal(got[0][0], got[1][0])
    # packs built afresh from the model's state give what the in-place writes gave
    model.invalidate_pack()
    for e, r in zip(both()[0], got[1]):
        assert torch.equal(e, r)
    model.undo_first_conv_restore()
    assert torch.equal(model.forward_batched(inputs, scales=scales)[1], before[1])


# ------------------------------------------------------------------------------------------------
# 3.-6. sample_requests
# ------------------------------------------------------------------------------------------------
def _att_masks(gi):
    from instancediffusion_b200 import ops
    counts = gi["masks"].sum(-1).round().int().contiguous()
    return ops.boxes_to_attmask(gi["boxes"].float().contiguous(), counts)


def _make_requests(unet, device):
    """The four requests of the issue, created so that the grounding input is last prepared at batch 1."""
    from instancediffusion_b200 import synthetic
    from instancediffusion_b200.ldm.models.diffusion.batched import Request
    from instancediffusion_b200.utils.model import alpha_generator
    gti = unet.grounding_tokenizer_input
    agen = partial(alpha_generator, type=[0.8, 0.0, 0.2])
    c_in, c_uc = synthetic.make_sampler_inputs(gti, 2, 3, 83, "box", mis=True, device=device)
    a_in, a_uc = synthetic.make_sampler_inputs(gti, 1, 2, 81, "box", mis=False, device=device)
    b_in, b_uc = synthetic.make_sampler_inputs(gti, 1, 1, 82, "box", mis=True, device=device)
    d_in, d_uc = synthetic.make_sampler_inputs(gti, 1, 5, 84, "box", mis=True, device=device)
    for inp in d_in:
        inp["grounding_input"]["att_masks"] = _att_masks(inp["grounding_input"])
    return [
        Request(input=a_in, uc=a_uc, guidance_scale=7.5, alpha_generator_func=agen, shape=(1, 4, 64, 64)),
        Request(input=b_in, uc=b_uc, guidance_scale=7.5, alpha_generator_func=agen, mis=0.36, shape=(1, 4, 64, 64)),
        Request(input=c_in, uc=c_uc, guidance_scale=7.5, alpha_generator_func=agen, mis=0.36, shape=(2, 4, 64, 64)),
        Request(input=d_in, uc=d_uc, guidance_scale=5.0, alpha_generator_func=partial(alpha_generator, type=[0.5, 0.0, 0.5]),
                mis=0.36, shape=(1, 4, 64, 64)),
    ]


def _fresh(req):
    """A copy of the request whose input dicts (and latents) the samplers may mutate."""
    from dataclasses import replace
    if isinstance(req.input, list):
        x = req.input[0]["x"].clone()
        return replace(req, input=[dict(i, x=x) for i in req.input])
    return replace(req, input=dict(req.input, x=req.input["x"].clone()))


def _run_alone(unet, diffusion, req, S):
    from instancediffusion_b200.ldm.models.diffusion.plms import PLMSSampler
    from instancediffusion_b200.ldm.models.diffusion.plms_instance import PLMSSamplerInst
    from instancediffusion_b200.utils.model import set_alpha_scale
    _reset(unet)
    req = _fresh(req)
    if isinstance(req.input, list):
        sampler = PLMSSamplerInst(diffusion, unet, alpha_generator_func=req.alpha_generator_func,
                                  set_alpha_scale=set_alpha_scale, mis=req.mis)
    else:
        sampler = PLMSSampler(diffusion, unet, alpha_generator_func=req.alpha_generator_func, set_alpha_scale=set_alpha_scale)
    out = sampler.sample(S=S, shape=req.shape, input=req.input, uc=req.uc, guidance_scale=req.guidance_scale).clone()
    _reset(unet)
    return out


def test_sample_requests_match_each_request_alone(cuda_device, unet, diffusion):
    from instancediffusion_b200.ldm.models.diffusion.batched import sample_requests
    reqs = _make_requests(unet, cuda_device)
    alone = [_run_alone(unet, diffusion, r, S_TEST) for r in reqs]
    _reset(unet)
    got = sample_requests(unet, diffusion, [_fresh(r) for r in reqs], S_TEST, max_batch=8)
    # the model is left as the sequential run of the same requests leaves it
    assert unet._first_conv_restored
    assert all(blk.fuser.scale == 0 for st in unet._transformers() for blk in st.transformer_blocks)
    _reset(unet)
    for k, (g, a) in enumerate(zip(got, alone)):
        r = _rel(g, a)
        print(f"[sample_requests] request {k}: rel_l2 vs its own sampler {r:.2e} (tol {LATENT_TOL:.1e})")
        assert r < LATENT_TOL, (k, r)


def test_sample_requests_schedule_longer_than_S(cuda_device, unet, diffusion):
    """S = 11 builds a 12-step schedule (range(0, 1000, 90)): a Multi-instance request merges before step
    int(12 * 0.36) = 4 as in PLMSSamplerInst, and with mis = 1 after the last step."""
    from instancediffusion_b200 import synthetic
    from instancediffusion_b200.ldm.models.diffusion.batched import Request, sample_requests
    from instancediffusion_b200.utils.model import alpha_generator
    gti = unet.grounding_tokenizer_input
    agen = partial(alpha_generator, type=[0.8, 0.0, 0.2])
    reqs = []
    for seed, n, mis in ((121, 2, 0.36), (122, 1, 1.0), (123, 3, 0.0)):
        inputs, uc = synthetic.make_sampler_inputs(gti, 1, n, seed, "box", mis=mis > 0, device=cuda_device)
        reqs.append(Request(input=inputs, uc=uc, guidance_scale=7.5, alpha_generator_func=agen, mis=mis,
                            shape=(1, 4, 64, 64)))
    alone = [_run_alone(unet, diffusion, r, 11) for r in reqs]
    _reset(unet)
    try:
        got = sample_requests(unet, diffusion, [_fresh(r) for r in reqs], 11)
    finally:
        _reset(unet)
    for k, (g, a) in enumerate(zip(got, alone)):
        r = _rel(g, a)
        print(f"[sample_requests S=11] request {k} (mis {reqs[k].mis}): rel_l2 vs its own sampler {r:.2e}")
        assert r < LATENT_TOL, (k, r)


def test_sample_requests_reference_anchor(cuda_device, unet, diffusion):
    """The samplers_extra mis_S10_n3 case (golden latent from the reference's own modules), batched together with an
    unrelated plain-PLMS request."""
    from instancediffusion_b200 import synthetic
    from instancediffusion_b200.ldm.models.diffusion.batched import Request, sample_requests
    from instancediffusion_b200.utils.model import alpha_generator
    gold = torch.load(os.path.join(GOLDEN, "samplers_extra.pt"), map_location="cpu")
    sc = cases.SAMPLER_EXTRA_CASES["mis_S10_n3"]
    gti = unet.grounding_tokenizer_input
    other, other_uc = synthetic.make_sampler_inputs(gti, 1, 4, 91, "box", mis=False, device=cuda_device)
    inputs, uc = synthetic.make_sampler_inputs(gti, sc["batch"], sc["n"], sc["seed"], "box", mis=True, device=cuda_device)
    reqs = [Request(input=other, uc=other_uc, guidance_scale=3.0,
                    alpha_generator_func=partial(alpha_generator, type=[0.3, 0.0, 0.7]), shape=(1, 4, 64, 64)),
            Request(input=inputs, uc=uc, guidance_scale=sc["guidance"],
                    alpha_generator_func=partial(alpha_generator, type=sc["alpha_type"]), mis=sc["mis"],
                    shape=(sc["batch"], 4, 64, 64))]
    _reset(unet)
    try:
        got = sample_requests(unet, diffusion, reqs, sc["S"])
    finally:
        _reset(unet)
    r = _rel(got[1], gold["mis_S10_n3"])
    print(f"[sample_requests] mis_S10_n3 next to another request: rel_l2 vs reference golden {r:.3e} (tol {LATENT_TOL:.1e})")
    assert r < LATENT_TOL, r


def test_sample_requests_new_alpha_pattern_reuses_graphs(cuda_device, unet, diffusion):
    from instancediffusion_b200 import synthetic
    from instancediffusion_b200.ldm.models.diffusion.batched import Request, sample_requests
    from instancediffusion_b200.utils.model import alpha_generator
    gti = unet.grounding_tokenizer_input
    ins = [synthetic.make_sampler_inputs(gti, 1, 2, s, "box", device=cuda_device) for s in (101, 102)]

    def reqs(types):
        return [Request(input=dict(i, x=i["x"].clone()), uc=uc, guidance_scale=7.5, shape=(1, 4, 64, 64),
                        alpha_generator_func=partial(alpha_generator, type=t)) for (i, uc), t in zip(ins, types)]
    unet.use_cuda_graph = True
    try:
        _reset(unet)
        sample_requests(unet, diffusion, reqs([[0.8, 0.0, 0.2], [0.6, 0.0, 0.4]]), S_TEST)
        n = len(unet._graphs)
        _reset(unet)
        sample_requests(unet, diffusion, reqs([[0.6, 0.0, 0.4], [0.8, 0.0, 0.2]]), S_TEST)
        assert len(unet._graphs) == n, (n, len(unet._graphs))
    finally:
        _reset(unet)


def test_sample_requests_rejects_mismatched_requests(cuda_device, unet, diffusion):
    from instancediffusion_b200 import synthetic
    from instancediffusion_b200.ldm.models.diffusion.batched import Request, sample_requests
    gti = unet.grounding_tokenizer_input
    a, uc = synthetic.make_sampler_inputs(gti, 1, 2, 111, "box", device=cuda_device)
    small, uc_s = synthetic.make_sampler_inputs(gti, 1, 2, 112, "box", device=cuda_device, size=48)
    ok = Request(input=a, uc=uc, guidance_scale=7.5)
    with pytest.raises(ValueError):
        sample_requests(unet, diffusion, [ok, Request(input=dict(a), uc=uc, guidance_scale=7.5, S=20)], S_TEST)
    with pytest.raises(ValueError):
        sample_requests(unet, diffusion, [ok, Request(input=small, uc=uc_s, guidance_scale=7.5)], S_TEST)
