"""`-m gpu` tests of DPM-Solver++(2M): the fused update (idiff_dpmpp2m_update) against float64 torch in both storage
builds, DPMSolverSampler on the seeded UNet against the float64 restatement of its loop (tests/cases_dpm.py) driven by
the same UNet, DPM-Solver++ requests next to PLMS and DDIM ones in `sample_requests` and `SamplingEngine` against each
request's own sampler, and bit-identity in batch-invariant mode."""
import os
import sys
from dataclasses import replace
from functools import partial

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import cases_dpm as CP  # noqa: E402
import cases_img2img as CI  # noqa: E402
from test_ddim_gpu import DDIM_LATENT_TOL, _rel, diffusion, unet  # noqa: E402,F401 (module fixtures)
from test_engine_gpu import _drive  # noqa: E402
from test_img2img_gpu import _alone as _alone_other  # noqa: E402
from test_requests_gpu import _fresh, _reset  # noqa: E402

pytestmark = pytest.mark.gpu
DTYPES = [torch.float16, torch.bfloat16]
ALPHA_TYPE = [0.8, 0.0, 0.2]
# DPMSolverSampler vs the restated loop on the same UNet: the sampler runs cond + uncond as one batch-2 forward, the
# restatement as two batch-1 forwards, so the eps round differently in the 16-bit storage and CFG 7.5 compounds it, as
# for the other samplers (test_img2img_gpu.TAIL_TOL).  bf16 keeps 3 fewer mantissa bits than fp16.  Measured on an H100
# over the three requests of test_sampler_matches_restated_loop: up to 5.19e-3 (fp16) and 4.07e-2 (bf16); the bounds
# are twice that.
TAIL_TOL = {torch.float16: 1.04e-2, torch.bfloat16: 8.14e-2}
# A request in a driver vs the same request alone: test_ddim_gpu.DDIM_LATENT_TOL (8.8e-3), the forwards' batch sizes
# differ and round differently.  Measured on an H100 over the six requests of _requests: up to 5.16e-3 (a DPM-Solver++
# request from x_init in the engine).


# ------------------------------------------------------------------------------------------------
# 1. the kernel
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("cfg", [False, True])
@pytest.mark.parametrize("prev", [False, True])
@pytest.mark.parametrize("n", [2 * 4 * 64 * 64 + 3, 4099, 1])
def test_dpmpp2m_update_against_float64(cuda_device, dtype, cfg, prev, n):
    from instancediffusion_b200 import ops
    from instancediffusion_b200.ldm.models.diffusion.dpm_solver import dpmpp2m_coefs
    g = torch.Generator().manual_seed(19)
    x, e_c, e_u, x0_prev = (torch.randn(n, generator=g).to(cuda_device) for _ in range(4))
    a_t, a_n = float(np.float32(0.30212)), float(np.float32(0.61768))
    coefs = dpmpp2m_coefs(a_t, a_n, 0.21 if prev else None)
    alpha_t, sigma_t, c_x, c_d, w_cur, w_prev = (float(np.float32(c)) for c in coefs[:6])  # what the kernel receives
    with ops.storage(dtype):
        x0_out, x_out = torch.empty_like(x), torch.empty_like(x)
        ops.dpmpp2m_update(x, e_c, e_u if cfg else None, 7.5, x0_prev if prev else None, alpha_t, sigma_t, c_x, c_d,
                           w_cur, w_prev, x0_out, x_out)
    x0_ref, x_ref = torch.empty_like(x, dtype=torch.float64), torch.empty_like(x, dtype=torch.float64)
    CP.dpmpp2m_update(x, e_c, e_u if cfg else None, 7.5, x0_prev if prev else None, alpha_t, sigma_t, c_x, c_d,
                      w_cur, w_prev, x0_ref, x_ref)
    r_x, r_0 = _rel(x_out, x_ref), _rel(x0_out, x0_ref)
    print(f"[dpmpp2m_update {dtype} cfg={cfg} prev={prev} n={n}] rel_l2 x {r_x:.2e}, x0 {r_0:.2e}")
    assert r_x <= 1e-6 and r_0 <= 1e-6, (r_x, r_0)


def test_dpmpp2m_update_rejects_bad_arguments(cuda_device):
    from instancediffusion_b200 import ops
    from instancediffusion_b200._lib import IdiffError
    x = torch.zeros(16, device=cuda_device)
    args = (0.5, 0.8, 1.1, -0.4, 1.5, -0.5)
    with pytest.raises(IdiffError):
        ops.dpmpp2m_update(x, x, None, 1.0, None, *args, None, torch.empty(8, device=cuda_device))
    with pytest.raises(IdiffError):
        ops.dpmpp2m_update(x, x, None, 1.0, torch.zeros(15, device=cuda_device), *args, None, torch.empty_like(x))
    with pytest.raises(IdiffError):
        ops.dpmpp2m_update(x, x.half(), None, 1.0, None, *args, None, torch.empty_like(x))
    with pytest.raises(IdiffError):
        ops.dpmpp2m_update(x, x, None, 1.0, None, 0.0, *args[1:], None, torch.empty_like(x))


# ------------------------------------------------------------------------------------------------
# 2. the sampler
# ------------------------------------------------------------------------------------------------
def _requests(unet, device, S=10):
    """DPM-Solver++ requests: plain (batch 1), image-to-image at 0.6 (batch 2 from a batch-1 x_init) and one without
    CFG; then a plain PLMS, a DDIM at eta 0.5 and an image-to-image PLMS request.  The batch-2 inputs are built first,
    so the grounding input is last prepared at batch 1."""
    from instancediffusion_b200 import synthetic
    from instancediffusion_b200.ldm.models.diffusion.batched import Request
    from instancediffusion_b200.utils.model import alpha_generator
    gti = unet.grounding_tokenizer_input
    agen = partial(alpha_generator, type=ALPHA_TYPE)
    b_in, b_uc = synthetic.make_sampler_inputs(gti, 2, 3, 802, "box", device=device)
    ins = [synthetic.make_sampler_inputs(gti, 1, 2, 800 + k, "box", device=device) for k in (1, 3, 4, 5, 6)]
    x_init = torch.randn((1, 4, 64, 64), generator=torch.Generator().manual_seed(8)).to(device)
    common = dict(guidance_scale=7.5, alpha_generator_func=agen, S=S)
    return [
        Request(input=ins[0][0], uc=ins[0][1], shape=(1, 4, 64, 64), sampler="dpmpp_2m", **common),
        Request(input=b_in, uc=b_uc, shape=(2, 4, 64, 64), sampler="dpmpp_2m", x_init=x_init, strength=0.6, seed=21,
                **common),
        Request(input=ins[1][0], uc=None, shape=(1, 4, 64, 64), sampler="dpmpp_2m",
                **dict(common, guidance_scale=1.0)),
        Request(input=ins[2][0], uc=ins[2][1], shape=(1, 4, 64, 64), **common),
        Request(input=ins[3][0], uc=ins[3][1], shape=(1, 4, 64, 64), sampler="ddim", eta=0.5, seed=22, **common),
        Request(input=ins[4][0], uc=ins[4][1], shape=(1, 4, 64, 64), x_init=x_init, strength=0.35, seed=23, **common),
    ]


def _alone(unet, diffusion, req):
    """The request through its own sampler, alone on the UNet."""
    from instancediffusion_b200.ldm.models.diffusion.dpm_solver import DPMSolverSampler
    from instancediffusion_b200.utils.model import set_alpha_scale
    if req.sampler != "dpmpp_2m":
        return _alone_other(unet, diffusion, req)
    _reset(unet)
    req = _fresh(req)
    s = DPMSolverSampler(diffusion, unet, alpha_generator_func=req.alpha_generator_func,
                         set_alpha_scale=set_alpha_scale)
    new = {} if req.x_init is None else dict(x_init=req.x_init, strength=req.strength, seed=req.seed)
    out = s.sample(S=req.S, shape=req.shape, input=req.input, uc=req.uc, guidance_scale=req.guidance_scale,
                   **new).clone()
    _reset(unet)
    return out


def _restated(unet, req):
    """cases_dpm's loop on the request, its eps from the same UNet one input at a time, the fuser scale and first conv
    set as the sampler sets them."""
    from instancediffusion_b200.utils.model import set_alpha_scale
    req = _fresh(req)
    _reset(unet)

    def eval_fn(inp, alpha):
        set_alpha_scale(unet, alpha)
        if alpha == 0:
            unet.restore_first_conv_from_SD()
        return unet(dict(inp)).float()
    if req.x_init is None:
        k0, xs = 0, req.input["x"]
    else:
        k0, xs = CI.start_latent(req.x_init, req.S, req.strength, req.seed, req.shape)
    try:
        return CP.dpm_tail(eval_fn, req.input, req.uc, req.S, req.guidance_scale, xs, k0, alpha_type=ALPHA_TYPE)
    finally:
        _reset(unet)


@pytest.mark.parametrize("dtype", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("k", [0, 1, 2])
def test_sampler_matches_restated_loop(cuda_device, unet, diffusion, dtype, k):
    from instancediffusion_b200 import ops
    with ops.storage(dtype):
        req = _requests(unet, cuda_device)[k]
        got = _alone(unet, diffusion, req)
        want = _restated(unet, req)
    r = _rel(got, want)
    print(f"[dpm sampler {k} strength {req.strength} cfg {req.guidance_scale} {dtype}] rel_l2 vs restated loop {r:.2e}")
    assert r < TAIL_TOL[dtype], r


# ------------------------------------------------------------------------------------------------
# 3. the request drivers
# ------------------------------------------------------------------------------------------------
def test_sample_requests_match_each_request_alone(cuda_device, unet, diffusion):
    from instancediffusion_b200.ldm.models.diffusion.batched import sample_requests
    reqs = _requests(unet, cuda_device)
    alone = [_alone(unet, diffusion, r) for r in reqs]
    _reset(unet)
    try:
        got = sample_requests(unet, diffusion, [_fresh(r) for r in reqs], 10, max_batch=8)
    finally:
        _reset(unet)
    for k, (g, a) in enumerate(zip(got, alone)):
        r = _rel(g, a)
        print(f"[sample_requests + dpm] request {k} ({reqs[k].sampler}, strength {reqs[k].strength}): "
              f"rel_l2 vs alone {r:.2e}")
        assert r < DDIM_LATENT_TOL, (k, r)


def test_engine_matches_each_request_alone(cuda_device, unet, diffusion):
    from instancediffusion_b200.ldm.models.diffusion.engine import SamplingEngine
    reqs = _requests(unet, cuda_device)
    reqs[0], reqs[3] = replace(reqs[0], S=20), replace(reqs[3], S=11)
    alone = [_alone(unet, diffusion, r) for r in reqs]
    _reset(unet)
    try:
        got = _drive(SamplingEngine(unet, diffusion, max_batch=8), reqs, [0, 0, 2, 3, 5, 6])
    finally:
        _reset(unet)
    for k, a in enumerate(alone):
        r = _rel(got[k], a)
        print(f"[engine + dpm] request {k} ({reqs[k].sampler}, S {reqs[k].S}): rel_l2 vs alone {r:.2e}")
        assert r < DDIM_LATENT_TOL, (k, r)


@pytest.mark.parametrize("dtype", DTYPES, ids=["fp16", "bf16"])
def test_batch_invariant_dpm_requests(cuda_device, unet, diffusion, dtype):
    """With batch-invariant mode on, DPM-Solver++ requests give the same bits alone, in sample_requests and in
    SamplingEngine, next to PLMS and DDIM requests."""
    from instancediffusion_b200 import ops
    from instancediffusion_b200.ldm.models.diffusion.batched import sample_requests
    from instancediffusion_b200.ldm.models.diffusion.engine import SamplingEngine
    with ops.storage(dtype):
        ops.set_batch_invariant(True)
        try:
            reqs = _requests(unet, cuda_device)
            targets = (0, 1, 2)
            alone = {j: _alone(unet, diffusion, reqs[j]) for j in targets}
            got = sample_requests(unet, diffusion, [_fresh(r) for r in reqs], 10, max_batch=8)
            _reset(unet)
            for j in targets:
                assert torch.equal(got[j], alone[j]), j
            got = _drive(SamplingEngine(unet, diffusion, max_batch=8, buckets=(2, 4, 8)), reqs, [0, 1, 0, 2, 0, 3])
            _reset(unet)
            for j in targets:
                assert torch.equal(got[j], alone[j]), j
        finally:
            ops.set_batch_invariant(False)
            _reset(unet)
