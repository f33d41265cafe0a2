"""`-m gpu` tests of DDIM sampling: the fused update (idiff_ddim_update) against float64 torch, its in-kernel noise
stream against the numpy mirror of tests/cases_ddim.py, DDIMSampler against the reference's latents
(tests/golden/ddim.pt), seeded repeatability at eta > 0, and DDIM requests next to PLMS ones in `sample_requests` and
`SamplingEngine`, with and without batch-invariant mode."""
import os
import sys
from dataclasses import replace
from functools import partial

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import cases_ddim as CD  # noqa: E402
from test_engine_gpu import _drive  # noqa: E402
from test_requests_gpu import _fresh, _reset, _run_alone  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(HERE, "golden")
DTYPES = [torch.float16, torch.bfloat16]
# DDIMSampler (fp16 storage) vs the reference's fp32 latent: 2x the measured relative L2 (H100: 4.48e-3 for ddim_S4,
# 3.39e-3 for ddim_S10_b2)
DDIM_GOLDEN_TOL = 9.0e-3
# A request in a driver vs the same request run alone, batch-invariant mode off: the forwards of the two runs have
# different batch sizes and so round differently at the fp16 level, and ten CFG-7.5 steps compound that.  Measured on
# an H100 over the mix of _mixed_requests: up to 4.41e-3 for a DDIM request and 4.38e-3 for the plain PLMS request,
# which sits at test_requests_gpu's LATENT_TOL (4.4e-3) too; the bound is 2x the measured maximum.  With the mode on,
# test_batch_invariant_ddim_request shows the two runs are bit-identical: the difference is the forwards' rounding.
DDIM_LATENT_TOL = 8.8e-3


def _rel(got, ref):
    got, ref = got.detach().double().cpu(), ref.detach().double().cpu()
    assert got.shape == ref.shape and torch.isfinite(got).all()
    return ((got - ref).norm() / ref.norm()).item()


def _noise(seed, index, n, device):
    """The kernel's z for (seed, index): x = 0, e_c = 0, no e_u, sigma = 1 -> x_out = z."""
    from instancediffusion_b200 import ops
    zero = torch.zeros(n, device=device)
    z = torch.empty(n, device=device)
    ops.ddim_update(zero, zero, None, 1.0, 0.5, 0.5, 1.0, seed, index, None, z)
    return z


# ------------------------------------------------------------------------------------------------
# 1. the kernel
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("cfg", [False, True])
@pytest.mark.parametrize("sigma", [0.0, 0.4])
def test_ddim_update_against_float64(cuda_device, dtype, cfg, sigma):
    from instancediffusion_b200 import ops
    n = 2 * 4 * 64 * 64 + 3  # a tail that does not fill a group of four
    g = torch.Generator().manual_seed(17)
    x, e_c, e_u = (torch.randn(n, generator=g).to(cuda_device) for _ in range(3))
    a_t, a_prev, gs, seed, index = 0.30212, 0.61768, 7.5, 2 ** 33 + 12345, 7
    a_t, a_prev = float(np.float32(a_t)), float(np.float32(a_prev))
    with ops.storage(dtype):
        e_out, x_out = torch.empty_like(x), torch.empty_like(x)
        ops.ddim_update(x, e_c, e_u if cfg else None, gs, a_t, a_prev, sigma, seed, index, e_out, x_out)
        z = _noise(seed, index, n, cuda_device).double()
    xd, ecd, eud = x.double(), e_c.double(), e_u.double()
    e = eud + gs * (ecd - eud) if cfg else ecd
    pred0 = (xd - (1 - a_t) ** 0.5 * e) / a_t ** 0.5
    ref = a_prev ** 0.5 * pred0 + (1 - a_prev - sigma ** 2) ** 0.5 * e + sigma * z
    r_x, r_e = _rel(x_out, ref), _rel(e_out, e)
    print(f"[ddim_update {dtype} cfg={cfg} sigma={sigma}] rel_l2 x {r_x:.2e}, e {r_e:.2e}")
    assert r_x <= 1e-6 and r_e <= 1e-6, (r_x, r_e)


def test_noise_is_independent_of_the_storage_build(cuda_device):
    from instancediffusion_b200 import ops
    z = {}
    for dtype in DTYPES:
        with ops.storage(dtype):
            z[dtype] = _noise(99, 4, 70001, cuda_device)
    assert torch.equal(z[torch.float16], z[torch.bfloat16])


def test_ddim_update_rejects_bad_arguments(cuda_device):
    from instancediffusion_b200 import ops
    from instancediffusion_b200._lib import IdiffError
    x = torch.zeros(16, device=cuda_device)
    with pytest.raises(IdiffError):
        ops.ddim_update(x, x, None, 1.0, 0.5, 0.5, 0.1, -1, 0, None, torch.empty_like(x))
    with pytest.raises(IdiffError):
        ops.ddim_update(x, x, None, 1.0, 0.5, 0.5, 0.1, 1, 0, None, torch.empty(8, device=cuda_device))
    with pytest.raises(IdiffError):
        ops.ddim_update(x, x, None, 1.0, 0.5, 0.5, -0.1, 1, 0, None, torch.empty_like(x))


# ------------------------------------------------------------------------------------------------
# 2. the noise stream
# ------------------------------------------------------------------------------------------------
def test_noise_matches_the_cpu_mirror(cuda_device):
    n = 1 << 18
    for seed, index in ((0, 0), (123456789, 9), (2 ** 64 - 1, 49)):
        z = _noise(seed, index, n, cuda_device).double().cpu().numpy()
        want = CD.ddim_noise(seed, index, n)
        err = np.abs(z - want).max()
        print(f"[noise seed={seed} index={index}] max abs err vs mirror {err:.2e}")
        assert err <= 1e-5, err


def test_noise_of_an_element_does_not_depend_on_the_length(cuda_device):
    full = _noise(31, 3, 1 << 16, cuda_device)
    for n in (1, 5, 4096, 4099, 40001):
        assert torch.equal(_noise(31, 3, n, cuda_device), full[:n]), n


def test_noise_statistics(cuda_device):
    n = 1 << 18
    z = _noise(5, 2, n, cuda_device).double()
    for other in (_noise(6, 2, n, cuda_device), _noise(5, 1, n, cuda_device)):
        c = torch.corrcoef(torch.stack([z, other.double()]))[0, 1].item()
        assert abs(c) < 0.01, c
    mean, var = z.mean().item(), z.var().item()
    print(f"[noise statistics] mean {mean:.2e} var {var:.4f}")
    assert abs(mean) < 5 / n ** 0.5 and abs(var - 1) < 0.01, (mean, var)


# ------------------------------------------------------------------------------------------------
# 3. DDIMSampler
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def unet(cuda_device):
    from instancediffusion_b200.weights import build_unet
    model = build_unet("box", cuda_device, seed=0)
    model._sd_conv = torch.load(os.path.join(GOLDEN, "sd15_first_conv.pt"), map_location="cpu")
    # the reference reads pretrained/SD_v1_5_input_conv_weight_bias.pth at alpha == 0; the same tensors are a fixture
    model.restore_first_conv_from_SD = lambda: (None if getattr(model, "_first_conv_restored", False)
                                                else model.set_sd_first_conv(model._sd_conv))
    model.restore_first_conv_from_SD()  # the SD1.5 weights are known from here on (the engine's per-image conv)
    model.undo_first_conv_restore()
    yield model
    model.use_cuda_graph = True


@pytest.fixture(scope="module")
def diffusion(cuda_device):
    from instancediffusion_b200.ldm.models.diffusion.ldm import LatentDiffusion
    return LatentDiffusion(linear_start=0.00085, linear_end=0.012, timesteps=1000).to(cuda_device)


def _ddim_alone(unet, diffusion, req, S):
    from instancediffusion_b200.ldm.models.diffusion.ddim import DDIMSampler
    from instancediffusion_b200.utils.model import set_alpha_scale
    _reset(unet)
    req = _fresh(req)
    sampler = DDIMSampler(diffusion, unet, alpha_generator_func=req.alpha_generator_func, set_alpha_scale=set_alpha_scale)
    out = sampler.sample(S=S, shape=req.shape, input=req.input, uc=req.uc, guidance_scale=req.guidance_scale,
                         eta=req.eta, seed=req.seed).clone()
    _reset(unet)
    return out


def _alone(unet, diffusion, req, S):
    return _ddim_alone(unet, diffusion, req, S) if req.sampler == "ddim" else _run_alone(unet, diffusion, req, S)


@pytest.mark.parametrize("name", list(CD.DDIM_CASES))
def test_ddim_sampler_vs_reference_golden(cuda_device, unet, diffusion, name):
    """DDIMSampler at eta = 0 against the reference's DDIMSampler (fp32 CPU), fp16 storage with fp32 accumulation
    compounded over S CFG-7.5 forwards.  The bound is 2x the measured relative L2, which is printed."""
    from instancediffusion_b200.ldm.models.diffusion.batched import Request
    from instancediffusion_b200.utils.model import alpha_generator
    path = os.path.join(GOLDEN, "ddim.pt")
    if not os.path.exists(path):
        pytest.skip("ddim.pt not generated")
    gold = torch.load(path, map_location="cpu")
    sc = CD.DDIM_CASES[name]
    unet.use_cuda_graph = True
    inp, uc = CD.ref_inputs_for(unet.grounding_tokenizer_input, name, device=cuda_device)
    req = Request(input=inp, uc=uc, guidance_scale=sc["guidance"], shape=(sc["batch"], 4, 64, 64), sampler="ddim",
                  alpha_generator_func=partial(alpha_generator, type=sc["alpha_type"]))
    x = _ddim_alone(unet, diffusion, req, sc["S"])
    r = _rel(x, gold[name])
    print(f"[ddim sampler] {name}: rel_l2 vs reference golden {r:.3e}")
    assert r < DDIM_GOLDEN_TOL, r


def test_ddim_sampler_seeded_repeatability(cuda_device, unet, diffusion):
    from instancediffusion_b200 import synthetic
    from instancediffusion_b200.ldm.models.diffusion.batched import Request
    from instancediffusion_b200.utils.model import alpha_generator
    inp, uc = synthetic.make_sampler_inputs(unet.grounding_tokenizer_input, 1, 2, 501, "box", device=cuda_device)
    req = Request(input=inp, uc=uc, guidance_scale=7.5, shape=(1, 4, 64, 64), sampler="ddim", eta=1.0, seed=42,
                  alpha_generator_func=partial(alpha_generator, type=[0.8, 0.0, 0.2]))
    a, b = _ddim_alone(unet, diffusion, req, 10), _ddim_alone(unet, diffusion, req, 10)
    assert torch.equal(a, b)
    c = _ddim_alone(unet, diffusion, replace(req, seed=43), 10)
    d = _ddim_alone(unet, diffusion, replace(req, eta=0.0), 10)
    assert _rel(c, a) > 1e-2 and _rel(d, a) > 1e-2


# ------------------------------------------------------------------------------------------------
# 4. the request drivers
# ------------------------------------------------------------------------------------------------
def _mixed_requests(unet, device, S=10):
    """DDIM at eta 0 (batch 1), DDIM at eta 0.5 (batch 2, explicit seed), plain PLMS and a Multi-instance PLMS request;
    the batch-2 inputs are built first, so the grounding input is last prepared at batch 1."""
    from instancediffusion_b200 import synthetic
    from instancediffusion_b200.ldm.models.diffusion.batched import Request
    from instancediffusion_b200.utils.model import alpha_generator
    gti = unet.grounding_tokenizer_input
    agen = partial(alpha_generator, type=[0.8, 0.0, 0.2])
    b_in, b_uc = synthetic.make_sampler_inputs(gti, 2, 3, 602, "box", device=device)
    a_in, a_uc = synthetic.make_sampler_inputs(gti, 1, 2, 601, "box", device=device)
    p_in, p_uc = synthetic.make_sampler_inputs(gti, 1, 2, 603, "box", device=device)
    m_in, m_uc = synthetic.make_sampler_inputs(gti, 1, 2, 604, "box", mis=True, device=device)
    return [
        Request(input=a_in, uc=a_uc, guidance_scale=7.5, alpha_generator_func=agen, shape=(1, 4, 64, 64), S=S,
                sampler="ddim"),
        Request(input=b_in, uc=b_uc, guidance_scale=5.0, alpha_generator_func=partial(alpha_generator, type=[0.5, 0.0, 0.5]),
                shape=(2, 4, 64, 64), S=S, sampler="ddim", eta=0.5, seed=2024),
        Request(input=p_in, uc=p_uc, guidance_scale=7.5, alpha_generator_func=agen, shape=(1, 4, 64, 64), S=S),
        Request(input=m_in, uc=m_uc, guidance_scale=7.5, alpha_generator_func=agen, mis=0.36, shape=(1, 4, 64, 64), S=S),
    ]


def test_sample_requests_with_ddim_match_each_request_alone(cuda_device, unet, diffusion):
    from instancediffusion_b200.ldm.models.diffusion.batched import sample_requests
    reqs = _mixed_requests(unet, cuda_device)
    alone = [_alone(unet, diffusion, r, 10) for r in reqs]
    _reset(unet)
    try:
        got = sample_requests(unet, diffusion, [_fresh(r) for r in reqs], 10, max_batch=8)
    finally:
        _reset(unet)
    for k, (g, a) in enumerate(zip(got, alone)):
        r = _rel(g, a)
        print(f"[sample_requests + DDIM] request {k} ({reqs[k].sampler}, eta {reqs[k].eta}): rel_l2 vs alone {r:.2e}")
        assert r < DDIM_LATENT_TOL, (k, r)


def test_engine_with_ddim_matches_each_request_alone(cuda_device, unet, diffusion):
    from instancediffusion_b200.ldm.models.diffusion.engine import SamplingEngine
    reqs = _mixed_requests(unet, cuda_device)
    reqs[1], reqs[2] = replace(reqs[1], S=11), replace(reqs[2], S=11)
    alone = [_alone(unet, diffusion, r, r.S) for r in reqs]
    _reset(unet)
    try:
        got = _drive(SamplingEngine(unet, diffusion, max_batch=8), reqs, [0, 2, 3, 5])
    finally:
        _reset(unet)
    for k, a in enumerate(alone):
        r = _rel(got[k], a)
        print(f"[engine + DDIM] request {k} ({reqs[k].sampler}, S {reqs[k].S}): rel_l2 vs alone {r:.2e}")
        assert r < DDIM_LATENT_TOL, (k, r)


@pytest.mark.parametrize("dtype", DTYPES, ids=["fp16", "bf16"])
def test_batch_invariant_ddim_request(cuda_device, unet, diffusion, dtype):
    """With batch-invariant mode on, an eta = 0.5 DDIM request gives the same bits alone, in sample_requests and in
    SamplingEngine, next to other requests."""
    from instancediffusion_b200 import ops
    from instancediffusion_b200.ldm.models.diffusion.batched import sample_requests
    from instancediffusion_b200.ldm.models.diffusion.engine import SamplingEngine
    with ops.storage(dtype):
        ops.set_batch_invariant(True)
        try:
            reqs = _mixed_requests(unet, cuda_device)
            target = replace(reqs[0], eta=0.5, seed=77)
            reqs = [reqs[2], target, reqs[1], reqs[3]]
            alone = _ddim_alone(unet, diffusion, target, 10)
            _reset(unet)
            got = sample_requests(unet, diffusion, [_fresh(r) for r in reqs], 10, max_batch=8)
            _reset(unet)
            assert torch.equal(got[1], alone)
            got = _drive(SamplingEngine(unet, diffusion, max_batch=8, buckets=(2, 4, 8)), reqs, [0, 1, 0, 2])
            _reset(unet)
            assert torch.equal(got[1], alone)
        finally:
            ops.set_batch_invariant(False)
            _reset(unet)
