"""Image-to-image sampling without a GPU: the start step of a strength, validation, the start latent, the three
samplers against the torch restatement of their loops from k0 (tests/cases_img2img.py), the unchanged path without
x_init, the seed draws, and image-to-image requests of several strengths next to plain PLMS / DDIM / Multi-instance
ones in `sample_requests` and `SamplingEngine`.  The UNet is the fake of fake_unet.py and the kernels are restated in
torch."""
import os
import sys
from dataclasses import replace

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import cases_img2img as CI  # noqa: E402
import cases_noise as CN  # noqa: E402
from fake_unet import FakeUNet, _fresh, _req, torch_kernels  # noqa: E402,F401
from instancediffusion_b200.ldm.models.diffusion._plms_common import PLMSBase  # noqa: E402
from instancediffusion_b200.ldm.models.diffusion.batched import (  # noqa: E402
    RequestPlan, _RequestState, check_requests, sample_requests, schedule_steps)
from instancediffusion_b200.ldm.models.diffusion.ddim import DDIMSampler  # noqa: E402
from instancediffusion_b200.ldm.models.diffusion.engine import SamplingEngine  # noqa: E402
from instancediffusion_b200.ldm.models.diffusion.plms import PLMSSampler  # noqa: E402
from instancediffusion_b200.ldm.models.diffusion.plms_instance import PLMSSamplerInst  # noqa: E402
from instancediffusion_b200.utils.model import set_alpha_scale  # noqa: E402

ALPHA_TYPE = [0.8, 0.0, 0.2]  # fake_unet.AGEN
TOL = dict(rtol=1e-5, atol=1e-6)


@pytest.fixture
def diffusion():
    from instancediffusion_b200.ldm.models.diffusion.ldm import LatentDiffusion
    return LatentDiffusion(linear_start=0.00085, linear_end=0.012, timesteps=1000)


def _x_init(seed, b=1, size=64):
    return torch.randn((b, 4, size, size), generator=torch.Generator().manual_seed(seed))


def _i2i(req, strength, seed, b=1):
    """The request from a random image latent at `strength`, its start noise keyed by `seed`."""
    return replace(req, x_init=_x_init(1000 + (seed or 0) % 997, b), strength=strength, seed=seed)


def _alone(diffusion, req, scale=0.0, model=None):
    """The request through its own sampler (PLMSSampler / PLMSSamplerInst / DDIMSampler) on a fresh fake."""
    model = FakeUNet(scale) if model is None else model
    req = _fresh(req)
    kw = dict(alpha_generator_func=req.alpha_generator_func, set_alpha_scale=set_alpha_scale)
    multi = isinstance(req.input, list)
    shape = (1, 4) + tuple((req.input[0] if multi else req.input)["x"].shape[2:])
    new = {} if req.x_init is None else dict(x_init=req.x_init, strength=req.strength, seed=req.seed)
    if req.sampler == "ddim":
        s = DDIMSampler(diffusion, model, **kw)
        new = dict(new, eta=req.eta, seed=req.seed)
    elif multi:
        s = PLMSSamplerInst(diffusion, model, mis=req.mis, **kw)
    else:
        s = PLMSSampler(diffusion, model, **kw)
    return s.sample(S=req.S, shape=shape, input=req.input, uc=req.uc, guidance_scale=req.guidance_scale, **new)


def _eval_fn():
    """FakeUNet's eps at fuser scale alpha, with the SD1.5 conv from the first alpha 0 on."""
    swapped = []

    def eval_fn(inp, alpha):
        swapped.append(alpha == 0)
        return (0.1 * inp["x"] + 1e-4 * inp["timesteps"].float().view(-1, 1, 1, 1) + 0.01 * inp["context"].mean()
                + 0.02 * float(alpha) + 0.03 * float(any(swapped)))
    return eval_fn


# ------------------------------------------------------------------------------------------------
# start step, validation, noise
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S", [10, 11, 50])
@pytest.mark.parametrize("strength", [0.01, 0.35, 0.999, 1.0])
def test_start_step(S, strength):
    N = schedule_steps(S)
    n_run = int(N * strength)
    if n_run == 0:
        with pytest.raises(ValueError, match="strength"):
            PLMSBase.start_step(N, strength)
        return
    k0 = PLMSBase.start_step(N, strength)
    assert k0 == N - n_run == CI.start_step(N, strength)
    assert {(10, 0.35): 7, (11, 0.35): 8, (50, 0.35): 33, (50, 0.999): 1, (11, 0.999): 1}.get((S, strength), k0) == k0
    if strength == 1.0:
        assert k0 == 0


def test_validation_messages(diffusion):
    s = PLMSSampler(diffusion, FakeUNet())
    inp = _req(1, 10).input
    with pytest.raises(ValueError, match="needs x_init"):
        s.sample(10, (1, 4, 64, 64), dict(inp), strength=0.5)
    for bad in (0.0, -0.2, 1.5, float("nan")):
        with pytest.raises(ValueError, match=r"outside \(0, 1\]"):
            s.sample(10, (1, 4, 64, 64), dict(inp), x_init=_x_init(1), strength=bad)
    with pytest.raises(ValueError, match="= 0 of the 10 steps"):
        s.sample(10, (1, 4, 64, 64), dict(inp), x_init=_x_init(1), strength=0.05)
    with pytest.raises(ValueError, match="does not fit the latent"):
        s.sample(10, (1, 4, 64, 64), dict(inp), x_init=_x_init(1, size=32), strength=0.5)
    with pytest.raises(ValueError, match="does not fit the latent"):
        s.sample(10, (2, 4, 64, 64), dict(inp), x_init=_x_init(1, b=3), strength=0.5)
    with pytest.raises(ValueError, match="needs x_init"):
        DDIMSampler(diffusion, FakeUNet()).sample(10, (1, 4, 64, 64), dict(inp), strength=0.5)

    ok = _req(2, 10)
    assert check_requests([_i2i(ok, 0.35, 1)], 10, 32) == [RequestPlan(1, None, 1, True, 7)]
    assert check_requests([_i2i(_req(3, 10, n=2, mis=0.36), 0.35, 1)], 10, 32) == [RequestPlan(1, None, 1, True, 7)]
    assert check_requests([_i2i(_req(3, 10, n=2, mis=0.36), 0.9, 1)], 10, 32) == [RequestPlan(3, 3, 1, True, 1)]
    with pytest.raises(ValueError, match="request 0: strength=0.5 needs x_init"):
        check_requests([replace(ok, strength=0.5)], 10, 32)
    with pytest.raises(ValueError, match=r"request 0: strength=1.5 outside"):
        check_requests([_i2i(ok, 1.5, 1)], 10, 32)
    with pytest.raises(ValueError, match="request 1: strength=0.05 runs"):
        check_requests([ok, _i2i(ok, 0.05, 1)], 10, 32)
    with pytest.raises(ValueError, match="request 0: x_init of shape"):
        check_requests([replace(ok, x_init=_x_init(1, size=32))], 10, 32)
    with pytest.raises(ValueError, match="inpainting"):  # still rejected with x_init
        check_requests([replace(_i2i(ok, 0.5, 1), mask=torch.zeros((1, 4, 64, 64)), x0=torch.zeros((1, 4, 64, 64)))],
                       10, 32)


def test_x_start64_noises_x_init_with_the_start_stream():
    x = CI.x_start64(torch.ones((1, 4, 2, 2)), 0.25, 7, (3, 4, 2, 2))
    want = 0.5 + 0.75 ** 0.5 * torch.from_numpy(CN.normals(7, CN.START, 0, 48)).view(3, 4, 2, 2)
    assert torch.allclose(x, want, rtol=0, atol=1e-15)


# ------------------------------------------------------------------------------------------------
# the samplers against the restated tail loops
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("strength", [0.35, 0.6, 1.0])
def test_plms_sampler_matches_restated_tail(diffusion, torch_kernels, strength):
    req = _i2i(_req(40, 10), strength, 11)
    got = _alone(diffusion, req)
    k0, xs = CI.start_latent(req.x_init, 10, strength, 11, (1, 4, 64, 64))
    want = CI.plms_tail(_eval_fn(), [_fresh(req).input], req.uc, 10, req.guidance_scale, xs, k0, alpha_type=ALPHA_TYPE)
    assert torch.allclose(got, want, **TOL)


@pytest.mark.parametrize("strength,merges", [(0.35, False), (0.9, True), (0.7, False), (0.8, True)])
def test_mis_sampler_matches_restated_tail(diffusion, torch_kernels, strength, merges):
    """mis 0.36 over 10 steps merges before step 3.  A run from k0 = 1 (0.9) or 2 (0.8) merges there; one from k0 = 3
    (0.7) or 7 (0.35) runs the global trajectory alone and calls no latent_mean."""
    req = _i2i(_req(41, 10, n=2, mis=0.36), strength, 12)
    k0, xs = CI.start_latent(req.x_init, 10, strength, 12, (1, 4, 64, 64))
    assert (3 > k0) == merges
    got = _alone(diffusion, req)
    assert torch_kernels["latent_mean"] == int(merges)
    want = CI.plms_tail(_eval_fn(), _fresh(req).input, req.uc, 10, req.guidance_scale, xs, k0, mis=0.36,
                        alpha_type=ALPHA_TYPE)
    assert torch.allclose(got, want, **TOL)


@pytest.mark.parametrize("eta", [0.0, 0.7])
@pytest.mark.parametrize("strength", [0.35, 0.6])
def test_ddim_sampler_matches_restated_tail(diffusion, torch_kernels, eta, strength):
    req = replace(_i2i(_req(42, 11), strength, 2 ** 40 + 3), sampler="ddim", eta=eta)
    got = _alone(diffusion, req)
    k0, xs = CI.start_latent(req.x_init, 11, strength, req.seed, (1, 4, 64, 64))
    want = CI.ddim_tail(_eval_fn(), _fresh(req).input, req.uc, 11, req.guidance_scale, xs, k0, eta=eta,
                        seed=req.seed, alpha_type=ALPHA_TYPE)
    assert torch.allclose(got, want, **TOL)


def test_x_init_broadcasts_over_the_batch(diffusion, torch_kernels):
    s = PLMSSampler(diffusion, FakeUNet())
    inp = dict(_req(43, 10).input, x=None)
    inp["context"] = inp["context"].expand(2, -1, -1)
    x0 = _x_init(5)
    s.sample(10, (2, 4, 64, 64), inp, x_init=x0, strength=1.0, seed=3)  # strength 1 from an image: k0 = 0
    assert inp["x"].shape == (2, 4, 64, 64)
    k0, xs = CI.start_latent(x0, 10, 1.0, 3, (2, 4, 64, 64))
    assert k0 == 0 and not torch.allclose(xs[0], xs[1])  # the batch's images are distinct variations


def test_without_x_init_every_sampler_is_unchanged(diffusion, torch_kernels):
    """x_init=None (strength 1) leaves each sampler's output bit-identical to a run without the new keywords."""
    cases = [_req(44, 10), _req(45, 10, n=2, mis=0.36), _req(46, 10, n=2, mis=0.0),
             replace(_req(47, 11), sampler="ddim", eta=0.7, seed=9)]
    for req in cases:
        a = _alone(diffusion, req)
        r = _fresh(req)
        multi = isinstance(r.input, list)
        kw = dict(alpha_generator_func=r.alpha_generator_func, set_alpha_scale=set_alpha_scale)
        if r.sampler == "ddim":
            s, extra = DDIMSampler(diffusion, FakeUNet(), **kw), dict(eta=r.eta, seed=r.seed)
        elif multi:
            s, extra = PLMSSamplerInst(diffusion, FakeUNet(), mis=r.mis, **kw), {}
        else:
            s, extra = PLMSSampler(diffusion, FakeUNet(), **kw), {}
        b = s.sample(S=r.S, shape=(1, 4, 64, 64), input=r.input, uc=r.uc, guidance_scale=r.guidance_scale,
                     x_init=None, strength=1.0, **extra)
        assert torch.equal(a, b)
    # mis 0 without x_init still merges (the identity in exact arithmetic) as before
    torch_kernels["latent_mean"] = 0
    _alone(diffusion, _req(46, 10, n=2, mis=0.0))
    assert torch_kernels["latent_mean"] == 1


def test_seed_draws(diffusion, torch_kernels):
    """An unseeded image-to-image run takes one draw from torch's default CPU generator (per sample call, or per request
    when it is constructed); runs without x_init draw what they drew before."""
    def draws(k):
        torch.manual_seed(99)
        return [int(torch.randint(0, 2 ** 63 - 1, (1,), dtype=torch.int64).item()) for _ in range(k)]
    want = draws(3)
    model = FakeUNet()
    s = PLMSSampler(diffusion, model)
    torch.manual_seed(99)
    s.sample(10, (1, 4, 64, 64), _fresh(_req(50, 10)).input, x_init=_x_init(1), strength=0.5)
    assert s.seed == want[0]
    reqs = [_i2i(_req(51, 10), 0.5, None), _req(52, 10), replace(_req(53, 10), sampler="ddim"),
            replace(_i2i(_req(54, 10), 0.5, None), sampler="ddim"), replace(_req(55, 10), sampler="ddim", eta=0.5)]
    plans = check_requests(reqs, 10, 32)
    torch.manual_seed(99)
    got = [_RequestState(r, p, 10, model, diffusion).base.seed for r, p in zip(reqs, plans)]
    assert got == [want[0], 0, 0, want[1], want[2]]
    torch.manual_seed(99)  # a seeded request draws nothing
    assert _RequestState(replace(reqs[0], seed=5), plans[0], 10, model, diffusion).base.seed == 5
    assert int(torch.randint(0, 2 ** 63 - 1, (1,), dtype=torch.int64).item()) == want[0]


# ------------------------------------------------------------------------------------------------
# the request drivers
# ------------------------------------------------------------------------------------------------
def _mix(S):
    """Plain PLMS, DDIM at eta 0.7, Multi-instance, and image-to-image PLMS / DDIM / MIS (merge after and at or
    before k0) requests at several strengths."""
    return [
        _req(60, S),
        replace(_req(61, S), sampler="ddim", eta=0.7, seed=1234),
        _req(62, S, n=2, mis=0.36),
        _i2i(_req(63, S), 0.35, 21),
        replace(_i2i(_req(64, S), 0.6, 22), sampler="ddim", eta=0.7),
        replace(_i2i(_req(65, S), 0.6, 23), sampler="ddim"),
        _i2i(_req(66, S, n=2, mis=0.36), 0.9, 24),
        _i2i(_req(67, S, n=3, mis=0.36, alpha=None), 0.35, 25),
    ]


def _images(req, S):
    """Images a request evaluates in a whole run: cond + uncond per live trajectory and step from k0, and the
    corrector's evaluation of a first PLMS step."""
    N = schedule_steps(S)
    k0 = 0 if req.x_init is None else N - int(N * req.strength)
    n = len(req.input) if isinstance(req.input, list) else 1
    merge = int(N * req.mis) if n > 1 else None
    if merge is not None and req.x_init is not None and merge <= k0:
        n, merge = 1, None

    def live(i):
        return n if merge is not None and i < merge else 1
    return 2 * (sum(live(i) for i in range(k0, N)) + (live(k0) if req.sampler == "plms" else 0))


@pytest.mark.parametrize("S", [10, 11])
def test_sample_requests_mixes_img2img_requests(diffusion, torch_kernels, S):
    reqs = _mix(S)
    model = FakeUNet(scale=0.5)
    got = sample_requests(model, diffusion, [_fresh(r) for r in reqs], S, max_batch=8)
    assert sum(sum(c["sizes"]) for c in model.calls) == sum(_images(r, S) for r in reqs)
    for k, r in enumerate(reqs):
        assert torch.allclose(got[k], _alone(diffusion, r, scale=0.5), **TOL), k


def test_engine_retires_img2img_after_n_run_ticks(diffusion, torch_kernels):
    for sampler, strength in (("plms", 0.35), ("ddim", 0.35), ("plms", 1.0), ("ddim", 0.6)):
        model = FakeUNet()
        eng = SamplingEngine(model, diffusion, buckets=None)
        req = replace(_i2i(_req(70, 11), strength, 31), sampler=sampler)
        finished, tick = {}, 0
        while tick <= 2 or eng.queued or eng.live:
            if tick == 2:
                eng.submit(_fresh(req))
            for t, x in eng.step().items():
                finished[t] = (tick, x)
            tick += 1
        N = schedule_steps(11)
        n_run = int(N * strength)
        ticks = n_run + (1 if sampler == "plms" else 0)
        assert finished[0][0] == 2 + ticks - 1 and len(model.calls) == ticks, (sampler, strength)
        assert torch.allclose(finished[0][1], _alone(diffusion, req), **TOL)


def test_engine_mixes_staggered_img2img_requests(diffusion, torch_kernels):
    model = FakeUNet()
    eng = SamplingEngine(model, diffusion, max_batch=8)
    mix = [replace(r, S=S) for r, S in zip(_mix(10), (10, 10, 11, 10, 20, 11, 10, 11))]
    arrivals = {0: mix[:3], 2: mix[3:5], 5: mix[5:7], 6: mix[7:]}
    out, reqs, tick, done_at, sub_at = {}, {}, 0, {}, {}
    while tick <= max(arrivals) or eng.queued or eng.live:
        for r in arrivals.get(tick, []):
            t = eng.submit(_fresh(r))
            reqs[t], sub_at[t] = r, tick
        for t, x in eng.step().items():
            out[t], done_at[t] = x, tick
        tick += 1
    assert set(out) == set(reqs)
    for t, r in reqs.items():
        assert torch.allclose(out[t], _alone(diffusion, r), **TOL), t
        N = schedule_steps(r.S)
        n_run = int(N * r.strength)
        assert done_at[t] - sub_at[t] + 1 == n_run + (r.sampler == "plms"), t  # admitted at once: live images fit
    evaluated = sum(sum(c["sizes"]) for c in model.calls) - eng.padded_images
    assert evaluated == sum(_images(r, r.S) for r in reqs.values())
