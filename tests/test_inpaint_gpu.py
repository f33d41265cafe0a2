"""`-m gpu` tests of inpainting requests: the blend kernel (idiff_inpaint_blend) against float64 and the numpy mirror of
its noise stream in both storage builds, its argument checks, inpainting requests through `sample_requests` against the
reference's own samplers with mask / x0 (tests/golden/inpaint.pt), the request drivers against each request's own
sampler with a seeded q_sample, bit-identity in batch-invariant mode, and one init_image -> inpaint -> image pass whose
unmasked bytes are the source's."""
import os
import sys
from contextlib import contextmanager
from dataclasses import replace
from functools import partial

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import cases  # noqa: E402
import cases_encode as CE  # noqa: E402
import cases_inpaint as CP  # noqa: E402
import cases_noise as CN  # noqa: E402
from test_ddim_gpu import DDIM_GOLDEN_TOL, DDIM_LATENT_TOL, _rel, diffusion, unet  # noqa: E402,F401 (module fixtures)
from test_engine_gpu import _drive  # noqa: E402
from test_requests_gpu import _fresh, _reset  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(HERE, "golden")
DTYPES = [torch.float16, torch.bfloat16]
ALPHA_TYPE = [0.8, 0.0, 0.2]
S = 10


# ------------------------------------------------------------------------------------------------
# 1. the kernel
# ------------------------------------------------------------------------------------------------
def _coefs(t):
    """(sqrt_a, sqrt_1m_a) of timestep t as the diffusion holds them (fp32 values)."""
    from instancediffusion_b200.ldm.models.diffusion.ldm import LatentDiffusion
    d = LatentDiffusion(linear_start=0.00085, linear_end=0.012, timesteps=1000)
    return float(d.sqrt_alphas_cumprod[t]), float(d.sqrt_one_minus_alphas_cumprod[t])


# (shape, x0 batch, keep batch, inputs as indices into the distinct tensors: repeats alias one input)
KERNEL_CASES = [
    ((1, 4, 64, 64), 1, 1, [0]),
    ((2, 4, 64, 64), 1, 2, [0, 0, 1]),   # aliased inputs, x0 broadcast
    ((8, 4, 64, 64), 8, 1, [0, 1, 2]),   # keep broadcast
    ((3, 3, 5, 7), 1, 3, [0, 1]),        # 315 elements: the last group of four is partial
]


@pytest.mark.parametrize("case", range(len(KERNEL_CASES)))
@pytest.mark.parametrize("seed,t", [(0, 981), (2 ** 64 - 1, 0), (123456789, 401)])
def test_inpaint_blend_against_float64(cuda_device, case, seed, t):
    """Kept elements against float64 (the noise of both builds rounded once to fp32), the others copied bit for bit;
    the fp16 and bf16 builds give the same bits."""
    from instancediffusion_b200 import ops
    shape, bx, bk, idx = KERNEL_CASES[case]
    g = torch.Generator().manual_seed(case)
    distinct = [torch.randn(shape, generator=g).to(cuda_device) for _ in range(max(idx) + 1)]
    xs = [distinct[i] for i in idx]
    x0 = torch.randn((bx,) + shape[1:], generator=g).to(cuda_device)
    keep = (torch.rand((bk,) + shape[2:], generator=g) < 0.6).to(torch.uint8).to(cuda_device)
    a = _coefs(t)
    got = {}
    for dtype in DTYPES:
        with ops.storage(dtype):
            outs = [torch.full(shape, float("nan"), device=cuda_device) for _ in xs]
            ops.inpaint_blend(xs, outs, x0, keep, a, seed, t)
            got[dtype] = [o.clone() for o in outs]
    for o16, ob in zip(got[torch.float16], got[torch.bfloat16]):
        assert torch.equal(o16, ob)
    want = CP.inpaint_blend64(xs, x0, keep, a, seed, t)
    k = keep.bool()[:, None].expand(shape).cpu()
    err = 0.0
    for o, w, x in zip(got[torch.float16], want, xs):
        o = o.cpu()
        assert torch.equal(o[~k], x.cpu()[~k])
        err = max(err, (o[k].double() - w[k]).abs().max().item())
    print(f"[inpaint_blend {shape} x0 {bx} keep {bk} count {len(xs)} seed={seed} t={t}] max abs err vs float64 "
          f"{err:.2e}")
    assert err <= 1e-5, err


def test_inpaint_blend_noise_matches_the_cpu_mirror(cuda_device):
    """x0 = 0, a = (0, 1), every element kept: the output is z itself."""
    from instancediffusion_b200 import ops
    n = 1 << 16
    shape = (1, 4, 128, 128)
    z = torch.empty(shape, device=cuda_device)
    ops.inpaint_blend([torch.zeros(shape, device=cuda_device)], [z], torch.zeros(shape, device=cuda_device),
                      torch.ones((1, 128, 128), dtype=torch.uint8, device=cuda_device), (0.0, 1.0), 77, 501)
    zz = z.double().cpu().reshape(-1).numpy()
    assert np.abs(zz - CN.normals(77, CN.INPAINT, 501, n)).max() <= 1e-5
    assert abs(zz.mean()) < 5 / n ** 0.5 and abs(zz.var() - 1) < 0.02


def test_inpaint_blend_rejects_bad_arguments(cuda_device):
    from instancediffusion_b200 import ops
    from instancediffusion_b200._lib import IdiffError
    dev = cuda_device
    x = torch.zeros((2, 4, 8, 8), device=dev)
    out = torch.empty_like(x)
    x0 = torch.zeros((1, 4, 8, 8), device=dev)
    keep = torch.ones((2, 8, 8), dtype=torch.uint8, device=dev)
    good = dict(xs=[x], outs=[out], x0=x0, keep=keep, a=(0.5, 0.5), seed=1, t=3)
    ops.inpaint_blend(**good)
    bad = [
        dict(outs=[out, torch.empty_like(x)]),                       # count mismatch
        dict(outs=[x]),                                              # in place
        dict(xs=[x, x], outs=[out, out]),                            # outputs alias each other
        dict(xs=[x.cpu()], outs=[out.cpu()]),                        # no CPU path
        dict(outs=[torch.empty((2, 4, 8, 9), device=dev)]),          # shape
        dict(xs=[x.half()]),                                         # dtype
        dict(x0=torch.zeros((2, 4, 8, 8), device=dev)[:, :, :, :8].transpose(2, 3)),  # non-contiguous
        dict(x0=torch.zeros((3, 4, 8, 8), device=dev)),              # x0 batch neither 1 nor B
        dict(x0=torch.zeros((1, 3, 8, 8), device=dev)),              # channels
        dict(keep=keep.bool()),                                      # dtype
        dict(keep=torch.ones((2, 1, 8, 8), dtype=torch.uint8, device=dev)),  # rank
        dict(keep=torch.ones((2, 8, 4), dtype=torch.uint8, device=dev)),
        dict(a=(1.5, 0.5)), dict(a=(0.5, -0.1)),
        dict(seed=-1), dict(seed=2 ** 64), dict(t=-1),
    ]
    for b in bad:
        with pytest.raises(IdiffError):
            ops.inpaint_blend(**dict(good, **b))


# ------------------------------------------------------------------------------------------------
# 2. requests against the reference and against their own samplers
# ------------------------------------------------------------------------------------------------
def _agen():
    from instancediffusion_b200.utils.model import alpha_generator
    return partial(alpha_generator, type=ALPHA_TYPE)


@pytest.mark.parametrize("name", list(CP.INPAINT_CASES))
def test_inpaint_requests_vs_reference_golden(cuda_device, unet, diffusion, name):
    """A strength-1 inpainting request through sample_requests against the reference's PLMSSampler / DDIMSampler with
    mask / x0 and the same seeded q_sample noise (fp32 CPU).  The bound is the DDIM golden's."""
    from instancediffusion_b200 import synthetic
    from instancediffusion_b200.ldm.models.diffusion.batched import Request, sample_requests
    from instancediffusion_b200.utils.model import alpha_generator
    gold = torch.load(os.path.join(GOLDEN, "inpaint.pt"), map_location="cpu")
    sc = CP.INPAINT_CASES[name]
    b = sc["batch"]
    unet.use_cuda_graph = True
    inp, uc = synthetic.make_sampler_inputs(unet.grounding_tokenizer_input, b, sc["n"], sc["input_seed"], "box",
                                            mis=False, device=cuda_device)
    x_init = torch.randn((b, 4, 64, 64), generator=torch.Generator().manual_seed(sc["src_seed"]))
    req = Request(input=inp, uc=uc, guidance_scale=sc["guidance"], shape=(b, 4, 64, 64), sampler=sc["sampler"],
                  alpha_generator_func=partial(alpha_generator, type=sc["alpha_type"]), x_init=x_init.to(cuda_device),
                  repaint_mask=CP.box_mask(1, 512, sc["box"]), seed=sc["seed"])
    _reset(unet)
    try:
        x = sample_requests(unet, diffusion, [req], sc["S"])[0]
    finally:
        _reset(unet)
    r = _rel(x, gold[name])
    print(f"[inpaint request] {name}: rel_l2 vs reference golden {r:.3e}")
    assert r < DDIM_GOLDEN_TOL, r


@contextmanager
def _seeded_q_sample(diffusion, seed):
    diffusion.q_sample = CP.seeded_q_sample(diffusion, seed)
    try:
        yield
    finally:
        del diffusion.q_sample


def _alone(unet, diffusion, req):
    """The request through its own sampler kind (`_sample`, or `sample_loop(mis=)` for a Multi-instance one) with mask
    = its keep mask, x0 = x_init over the batch and `diffusion.q_sample` drawing the seeded blend noise."""
    from instancediffusion_b200.ldm.models.diffusion.ddim import DDIMSampler
    from instancediffusion_b200.ldm.models.diffusion.dpm_solver import DPMSolverSampler
    from instancediffusion_b200.ldm.models.diffusion.plms import PLMSSampler
    from instancediffusion_b200.ldm.models.diffusion.plms_instance import PLMSSamplerInst
    from instancediffusion_b200.utils.model import set_alpha_scale
    _reset(unet)
    req = _fresh(req)
    multi = isinstance(req.input, list)
    kind = {"ddim": DDIMSampler, "dpmpp_2m": DPMSolverSampler}.get(req.sampler, PLMSSamplerInst if multi else PLMSSampler)
    s = kind(diffusion, unet, alpha_generator_func=req.alpha_generator_func, set_alpha_scale=set_alpha_scale)
    mask = x0 = None
    if req.repaint_mask is not None:
        mask = CP.keep_of(req.repaint_mask.cpu()).float()[:, None].to(req.x_init.device)
        x0 = req.x_init.expand(req.shape)
    try:
        with _seeded_q_sample(diffusion, req.seed):
            return s._sample(req.S, req.shape, req.input, req.uc, req.guidance_scale, mask, x0, req.x_init,
                             req.strength, req.seed, eta=req.eta, mis=req.mis if multi else None).clone()
    finally:
        _reset(unet)


def _requests(unet, device):
    """Inpainting PLMS (strength 1), DDIM at eta 0.7 (batch 2 from a batch-1 source and mask, strength 0.8),
    DPM-Solver++ (0.6) and Multi-instance PLMS (strength 1, merges at step 3), next to a plain PLMS request and an
    image-to-image DDIM one; the batch-2 inputs are built first, so the grounding input is last prepared at batch 1."""
    from instancediffusion_b200 import synthetic
    from instancediffusion_b200.ldm.models.diffusion.batched import Request
    gti = unet.grounding_tokenizer_input
    b_in, b_uc = synthetic.make_sampler_inputs(gti, 2, 3, 802, "box", device=device)
    ins = [synthetic.make_sampler_inputs(gti, 1, 2, 800 + k, "box", mis=k == 4, device=device) for k in (1, 3, 4, 5, 6)]

    def src(seed, b=1):
        return torch.randn((b, 4, 64, 64), generator=torch.Generator().manual_seed(seed)).to(device)
    box = CP.box_mask(1, 512, (96, 352, 128, 416))
    common = dict(guidance_scale=7.5, alpha_generator_func=_agen(), S=S, shape=(1, 4, 64, 64))
    return [
        Request(input=ins[0][0], uc=ins[0][1], x_init=src(1), repaint_mask=box, seed=11, **common),
        Request(input=b_in, uc=b_uc, **dict(common, shape=(2, 4, 64, 64)), sampler="ddim", eta=0.7, x_init=src(2),
                strength=0.8, repaint_mask=box.to(torch.uint8).to(device), seed=12),
        Request(input=ins[1][0], uc=ins[1][1], sampler="dpmpp_2m", x_init=src(3), strength=0.6,
                repaint_mask=CP.box_mask(1, 512, (0, 512, 256, 512)), seed=13, **common),
        Request(input=ins[2][0], uc=ins[2][1], mis=0.36, x_init=src(4), repaint_mask=box, seed=14, **common),
        Request(input=ins[3][0], uc=ins[3][1], **common),
        Request(input=ins[4][0], uc=ins[4][1], sampler="ddim", eta=0.5, x_init=src(5), strength=0.6, seed=15, **common),
    ]


def test_sample_requests_match_each_request_alone(cuda_device, unet, diffusion):
    from instancediffusion_b200.ldm.models.diffusion.batched import sample_requests
    reqs = _requests(unet, cuda_device)
    alone = [_alone(unet, diffusion, r) for r in reqs]
    _reset(unet)
    try:
        got = sample_requests(unet, diffusion, [_fresh(r) for r in reqs], S, max_batch=8)
    finally:
        _reset(unet)
    for k, (g, a) in enumerate(zip(got, alone)):
        r = _rel(g, a)
        print(f"[sample_requests + inpaint] request {k} ({reqs[k].sampler}, mask {reqs[k].repaint_mask is not None}): "
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
        print(f"[engine + inpaint] request {k} ({reqs[k].sampler}, S {reqs[k].S}): rel_l2 vs alone {r:.2e}")
        assert r < DDIM_LATENT_TOL, (k, r)


@pytest.mark.parametrize("dtype", DTYPES, ids=["fp16", "bf16"])
def test_batch_invariant_inpaint_requests(cuda_device, unet, diffusion, dtype):
    """With batch-invariant mode on, the PLMS, DDIM (eta 0.7) and Multi-instance inpainting requests give the same bits
    alone, in sample_requests next to the others and in SamplingEngine with graphs."""
    from instancediffusion_b200 import ops
    from instancediffusion_b200.ldm.models.diffusion.batched import sample_requests
    from instancediffusion_b200.ldm.models.diffusion.engine import SamplingEngine
    with ops.storage(dtype):
        ops.set_batch_invariant(True)
        try:
            reqs = _requests(unet, cuda_device)
            targets = (0, 1, 3)
            alone = {}
            for j in targets:
                _reset(unet)
                alone[j] = sample_requests(unet, diffusion, [_fresh(reqs[j])], S)[0]
            _reset(unet)
            got = sample_requests(unet, diffusion, [_fresh(r) for r in reqs], S, max_batch=8)
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
# 3. end to end through the first stage
# ------------------------------------------------------------------------------------------------
def test_init_image_inpaint_to_image(cuda_device, unet, diffusion):
    """A 512x512 image, a box repaint mask and output="image" in both drivers: every byte outside the box is the
    source's, the box is regenerated."""
    from oracle import torch_oracle as TO
    from instancediffusion_b200.ldm.models.autoencoder import AutoencoderKL
    from instancediffusion_b200.ldm.models.diffusion.engine import SamplingEngine
    from instancediffusion_b200.ldm.models.diffusion.batched import sample_requests
    from instancediffusion_b200.weights import synth_tensor
    with torch.device("meta"):
        vae = AutoencoderKL(dict(TO.VAE_DDCONFIG), 4, TO.VAE_SCALE)
    vae = vae.to_empty(device=cuda_device).eval()
    vae.load_state_dict({k: synth_tensor("vae." + k, tuple(v.shape), cases.WEIGHT_SEED)
                         for k, v in vae.state_dict().items()}, strict=True)
    src = CE.random_images(1, 512, 512, 8).to(cuda_device)
    box = CP.box_mask(1, 512, (100, 300, 60, 333))
    reqs = _requests(unet, cuda_device)
    req = replace(reqs[0], x_init=None, init_image=src, repaint_mask=box, output="image")
    _reset(unet)
    try:
        outs = [sample_requests(unet, diffusion, [_fresh(req), _fresh(reqs[4])], S, autoencoder=vae)[0]]
        _reset(unet)
        outs.append(_drive(SamplingEngine(unet, diffusion, max_batch=8, autoencoder=vae), [req], [0])[0])
    finally:
        _reset(unet)
    rep = box.to(cuda_device)[..., None].expand(1, 512, 512, 3)
    for img in outs:
        assert img.dtype == torch.uint8 and img.shape == (1, 512, 512, 3)
        assert torch.equal(img[~rep], src[~rep])
        changed = (img[rep] != src[rep]).float().mean().item()
        print(f"[inpaint to image] bytes changed inside the box: {changed:.3f}")
        assert changed > 0.5
