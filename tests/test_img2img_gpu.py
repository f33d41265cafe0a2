"""`-m gpu` tests of image-to-image sampling: the start-latent kernel (idiff_noise_latent) against float64 and the numpy
mirror of its noise stream in both storage builds, the three samplers on the seeded UNet against the torch restatement
of their loops from k0 (tests/cases_img2img.py) driven by the same UNet, seeded repeatability, both request drivers
against each request's own `sample()`, bit-identity in batch-invariant mode, CUDA-graph replay against eager, and one
encode -> image-to-image -> decode pass through the first stage."""
import os
import sys
from dataclasses import replace
from functools import partial

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import cases  # noqa: E402
import cases_img2img as CI  # noqa: E402
import cases_noise as CN  # noqa: E402
from test_ddim_gpu import DDIM_LATENT_TOL, _rel, diffusion, unet  # noqa: E402,F401 (module fixtures)
from test_engine_gpu import _drive  # noqa: E402
from test_requests_gpu import _fresh, _reset  # noqa: E402

pytestmark = pytest.mark.gpu
DTYPES = [torch.float16, torch.bfloat16]
ALPHA_TYPE = [0.8, 0.0, 0.2]
# A sampler's latent vs the restated loop on the same UNet: the sampler runs cond + uncond as one batch-2 forward, the
# restatement as two batch-1 forwards, so the eps round differently in the 16-bit storage and CFG 7.5 compounds it, as
# in test_ddim_gpu (DDIM_LATENT_TOL).  bf16 keeps 3 fewer mantissa bits than fp16.  Measured on an H100: up to 5.36e-3
# (fp16) and 4.16e-2 (bf16) over the four requests of test_sampler_matches_restated_tail.
TAIL_TOL = {torch.float16: DDIM_LATENT_TOL, torch.bfloat16: 8 * DDIM_LATENT_TOL}


def _x_init(seed, b, device):
    return torch.randn((b, 4, 64, 64), generator=torch.Generator().manual_seed(seed)).to(device)


# ------------------------------------------------------------------------------------------------
# 1. the kernel
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("shape,init", [((2, 4, 64, 64), (2, 4, 64, 64)), ((3, 4, 5, 7), (1, 4, 5, 7)),
                                        ((3, 1, 1, 1365), (1, 1, 1, 1365)), ((1, 1, 1, 4099), (1, 1, 1, 4099))])
@pytest.mark.parametrize("seed", [0, 2 ** 64 - 1, 123456789])
def test_noise_latent_against_float64(cuda_device, dtype, shape, init, seed):
    """Odd n (4095, 4099: the last group of four is partial), n_init < n (x_init broadcast over the batch)."""
    from instancediffusion_b200 import ops
    x_init = torch.randn(init, generator=torch.Generator().manual_seed(5)).to(cuda_device)
    a = float(np.float32(0.30212))
    with ops.storage(dtype):
        out = ops.noise_latent(x_init, a, seed, torch.empty(shape, device=cuda_device))
    want = CI.x_start64(x_init, a, seed, shape)
    err = (out.double().cpu() - want).abs().max().item()
    print(f"[noise_latent {dtype} {shape} seed={seed}] max abs err vs float64 {err:.2e}")
    assert err <= 1e-5, err


def test_noise_latent_is_z_at_a_0_and_independent_of_the_build(cuda_device):
    from instancediffusion_b200 import ops
    n = 1 << 16
    z = {}
    for dtype in DTYPES:
        with ops.storage(dtype):
            z[dtype] = ops.noise_latent(torch.zeros(n, device=cuda_device), 0.0, 77, torch.empty(n, device=cuda_device))
    assert torch.equal(z[torch.float16], z[torch.bfloat16])
    zz = z[torch.float16].double().cpu()
    assert np.abs(zz.numpy() - CN.normals(77, CN.START, 0, n)).max() <= 1e-5
    assert abs(zz.mean().item()) < 5 / n ** 0.5 and abs(zz.var().item() - 1) < 0.02


def test_noise_latent_rejects_bad_arguments(cuda_device):
    from instancediffusion_b200 import ops
    from instancediffusion_b200._lib import IdiffError
    x = torch.zeros(12, device=cuda_device)
    with pytest.raises(IdiffError):
        ops.noise_latent(x, 0.5, -1, torch.empty(12, device=cuda_device))
    with pytest.raises(IdiffError):
        ops.noise_latent(x, 0.5, 2 ** 64, torch.empty(12, device=cuda_device))
    with pytest.raises(IdiffError):
        ops.noise_latent(x, 0.5, 1, torch.empty(18, device=cuda_device))  # 18 % 12 != 0
    with pytest.raises(IdiffError):
        ops.noise_latent(x, 1.5, 1, torch.empty(24, device=cuda_device))
    with pytest.raises(IdiffError):
        ops.noise_latent(torch.zeros((4, 6), device=cuda_device)[:, :3], 0.5, 1, torch.empty(24, device=cuda_device))


# ------------------------------------------------------------------------------------------------
# 2. the samplers
# ------------------------------------------------------------------------------------------------
def _requests(unet, device, S=10):
    """Image-to-image PLMS (0.6), DDIM at eta 0.7 (0.35, batch 2 from a batch-1 x_init), Multi-instance (0.9: merges
    after k0) and Multi-instance (0.35: global trajectory alone), plus plain PLMS and DDIM requests; the batch-2 inputs
    are built first, so the grounding input is last prepared at batch 1."""
    from instancediffusion_b200 import synthetic
    from instancediffusion_b200.ldm.models.diffusion.batched import Request
    from instancediffusion_b200.utils.model import alpha_generator
    gti = unet.grounding_tokenizer_input
    agen = partial(alpha_generator, type=ALPHA_TYPE)
    b_in, b_uc = synthetic.make_sampler_inputs(gti, 2, 3, 702, "box", device=device)
    ins = [synthetic.make_sampler_inputs(gti, 1, 2, 700 + k, "box", mis=k in (3, 4), device=device)
           for k in (1, 3, 4, 5, 6)]
    common = dict(guidance_scale=7.5, alpha_generator_func=agen, S=S)
    return [
        Request(input=ins[0][0], uc=ins[0][1], shape=(1, 4, 64, 64), x_init=_x_init(1, 1, device), strength=0.6,
                seed=11, **common),
        Request(input=b_in, uc=b_uc, shape=(2, 4, 64, 64), sampler="ddim", eta=0.7, x_init=_x_init(2, 1, device),
                strength=0.35, seed=12, **common),
        Request(input=ins[1][0], uc=ins[1][1], shape=(1, 4, 64, 64), mis=0.36, x_init=_x_init(3, 1, device),
                strength=0.9, seed=13, **common),
        Request(input=ins[2][0], uc=ins[2][1], shape=(1, 4, 64, 64), mis=0.36, x_init=_x_init(4, 1, device),
                strength=0.35, seed=14, **common),
        Request(input=ins[3][0], uc=ins[3][1], shape=(1, 4, 64, 64), **common),
        Request(input=ins[4][0], uc=ins[4][1], shape=(1, 4, 64, 64), sampler="ddim", eta=0.5, seed=15, **common),
    ]


def _alone(unet, diffusion, req, S=None):
    from instancediffusion_b200.ldm.models.diffusion.ddim import DDIMSampler
    from instancediffusion_b200.ldm.models.diffusion.plms import PLMSSampler
    from instancediffusion_b200.ldm.models.diffusion.plms_instance import PLMSSamplerInst
    from instancediffusion_b200.utils.model import set_alpha_scale
    _reset(unet)
    req = _fresh(req)
    kw = dict(alpha_generator_func=req.alpha_generator_func, set_alpha_scale=set_alpha_scale)
    new = dict(x_init=req.x_init, strength=req.strength, seed=req.seed)
    if req.sampler == "ddim":
        s, new = DDIMSampler(diffusion, unet, **kw), dict(new, eta=req.eta)
    elif isinstance(req.input, list):
        s = PLMSSamplerInst(diffusion, unet, mis=req.mis, **kw)
    else:
        s = PLMSSampler(diffusion, unet, **kw)
    out = s.sample(S=S or req.S, shape=req.shape, input=req.input, uc=req.uc, guidance_scale=req.guidance_scale,
                   **new).clone()
    _reset(unet)
    return out


def _restated(unet, req):
    """cases_img2img's tail loop on the request, its eps from the same UNet one input at a time, the fuser scale and
    first conv set as the sampler sets them."""
    from instancediffusion_b200.utils.model import set_alpha_scale
    req = _fresh(req)
    _reset(unet)

    def eval_fn(inp, alpha):
        set_alpha_scale(unet, alpha)
        if alpha == 0:
            unet.restore_first_conv_from_SD()
        return unet(dict(inp)).float()
    k0, xs = CI.start_latent(req.x_init, req.S, req.strength, req.seed, req.shape)
    try:
        if req.sampler == "ddim":
            return CI.ddim_tail(eval_fn, req.input, req.uc, req.S, req.guidance_scale, xs, k0, eta=req.eta,
                                seed=req.seed, alpha_type=ALPHA_TYPE)
        ins = req.input if isinstance(req.input, list) else [req.input]
        return CI.plms_tail(eval_fn, ins, req.uc, req.S, req.guidance_scale, xs, k0, mis=req.mis,
                            alpha_type=ALPHA_TYPE)
    finally:
        _reset(unet)


@pytest.mark.parametrize("dtype", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("k", [0, 1, 2, 3])
def test_sampler_matches_restated_tail(cuda_device, unet, diffusion, dtype, k):
    from instancediffusion_b200 import ops
    with ops.storage(dtype):
        req = _requests(unet, cuda_device)[k]
        got = _alone(unet, diffusion, req)
        want = _restated(unet, req)
    r = _rel(got, want)
    print(f"[img2img sampler {k} {req.sampler} strength {req.strength} {dtype}] rel_l2 vs restated loop {r:.2e}")
    assert r < TAIL_TOL[dtype], r


def test_seeded_repeatability(cuda_device, unet, diffusion):
    req = _requests(unet, cuda_device)[0]
    a, b = _alone(unet, diffusion, req), _alone(unet, diffusion, req)
    assert torch.equal(a, b)
    c = _alone(unet, diffusion, replace(req, seed=req.seed + 1))
    d = _alone(unet, diffusion, replace(req, strength=0.35))
    assert _rel(c, a) > 1e-2 and _rel(d, a) > 1e-2
    # the start latent is the image's at low noise: strength 0.1 of 50 steps stays near x_init
    low = _alone(unet, diffusion, replace(req, strength=0.1, S=50))
    assert _rel(low, req.x_init) < _rel(_alone(unet, diffusion, replace(req, strength=1.0, S=50)), req.x_init)


def test_cuda_graph_replay_equals_eager(cuda_device, unet, diffusion):
    req = _requests(unet, cuda_device)[0]
    unet.use_cuda_graph = False
    try:
        eager = _alone(unet, diffusion, req)
    finally:
        unet.use_cuda_graph = True
    _alone(unet, diffusion, req)  # capture
    assert torch.equal(_alone(unet, diffusion, req), eager)


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
        print(f"[sample_requests + img2img] request {k} ({reqs[k].sampler}, strength {reqs[k].strength}): "
              f"rel_l2 vs alone {r:.2e}")
        assert r < DDIM_LATENT_TOL, (k, r)


def test_engine_matches_each_request_alone(cuda_device, unet, diffusion):
    from instancediffusion_b200.ldm.models.diffusion.engine import SamplingEngine
    reqs = _requests(unet, cuda_device)
    reqs[1], reqs[4] = replace(reqs[1], S=11), replace(reqs[4], S=11)
    alone = [_alone(unet, diffusion, r) for r in reqs]
    _reset(unet)
    try:
        got = _drive(SamplingEngine(unet, diffusion, max_batch=8), reqs, [0, 0, 2, 3, 5, 6])
    finally:
        _reset(unet)
    for k, a in enumerate(alone):
        r = _rel(got[k], a)
        print(f"[engine + img2img] request {k} ({reqs[k].sampler}, strength {reqs[k].strength}): rel_l2 vs alone {r:.2e}")
        assert r < DDIM_LATENT_TOL, (k, r)


@pytest.mark.parametrize("dtype", DTYPES, ids=["fp16", "bf16"])
def test_batch_invariant_img2img_requests(cuda_device, unet, diffusion, dtype):
    """With batch-invariant mode on, image-to-image requests give the same bits alone, in sample_requests and in
    SamplingEngine, next to other requests of other strengths."""
    from instancediffusion_b200 import ops
    from instancediffusion_b200.ldm.models.diffusion.batched import sample_requests
    from instancediffusion_b200.ldm.models.diffusion.engine import SamplingEngine
    with ops.storage(dtype):
        ops.set_batch_invariant(True)
        try:
            reqs = _requests(unet, cuda_device)
            targets = (0, 1, 3)
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


# ------------------------------------------------------------------------------------------------
# 4. end to end through the first stage
# ------------------------------------------------------------------------------------------------
def test_encode_img2img_decode(cuda_device, unet, diffusion):
    """A 512x512 image encoded by the seeded VAE, refined at strength 0.35 and decoded."""
    from oracle import torch_oracle as TO
    from instancediffusion_b200.ldm.models.autoencoder import AutoencoderKL
    from instancediffusion_b200.weights import synth_tensor
    with torch.device("meta"):
        vae = AutoencoderKL(dict(TO.VAE_DDCONFIG), 4, TO.VAE_SCALE)
    vae = vae.to_empty(device=cuda_device).eval()
    vae.load_state_dict({k: synth_tensor("vae." + k, tuple(v.shape), cases.WEIGHT_SEED)
                         for k, v in vae.state_dict().items()}, strict=True)
    img = torch.rand((1, 3, 512, 512), generator=torch.Generator().manual_seed(8)).to(cuda_device) * 2 - 1
    torch.manual_seed(0)
    with torch.no_grad():
        z = vae.encode(img)
    assert z.shape == (1, 4, 64, 64) and torch.isfinite(z).all()
    req = replace(_requests(unet, cuda_device)[0], x_init=z.float(), strength=0.35)
    lat = _alone(unet, diffusion, req)
    out = vae.decode(lat)
    assert lat.shape == (1, 4, 64, 64) and out.shape == (1, 3, 512, 512)
    assert torch.isfinite(lat).all() and torch.isfinite(out).all()
