"""Inpainting requests (`Request.repaint_mask`) without a GPU: validation, the pixel-to-latent mask reduction,
inpainting requests of every sampler kind next to plain and image-to-image requests in `sample_requests` and
`SamplingEngine` against each request's own sampler with `diffusion.q_sample` drawing the seeded blend noise, the
all-repaint / all-keep edges, the corrector of a first PLMS step, and the paste-back of image outputs.  The UNet is the
fake of fake_unet.py, the first stage the fake of cases_encode.py and the kernels are restated in torch."""
import os
import sys
from contextlib import contextmanager
from dataclasses import replace

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import cases_encode as CE  # noqa: E402
import cases_img2img as CI  # noqa: E402
import cases_inpaint as CP  # noqa: E402
from fake_unet import FakeUNet, _fresh, _req, torch_kernels  # noqa: E402,F401
from instancediffusion_b200.ldm.models.diffusion.batched import (  # noqa: E402
    check_requests, keep_mask, sample_requests)
from instancediffusion_b200.ldm.models.diffusion.ddim import DDIMSampler  # noqa: E402
from instancediffusion_b200.ldm.models.diffusion.dpm_solver import DPMSolverSampler  # noqa: E402
from instancediffusion_b200.ldm.models.diffusion.engine import SamplingEngine  # noqa: E402
from instancediffusion_b200.ldm.models.diffusion.plms import PLMSSampler  # noqa: E402
from instancediffusion_b200.ldm.models.diffusion.plms_instance import PLMSSamplerInst  # noqa: E402
from instancediffusion_b200.utils.model import set_alpha_scale  # noqa: E402

S = 10


@pytest.fixture
def diffusion():
    from instancediffusion_b200.ldm.models.diffusion.ldm import LatentDiffusion
    return LatentDiffusion(linear_start=0.00085, linear_end=0.012, timesteps=1000)


def _x_init(seed, b=1):
    return torch.randn((b, 4, 64, 64), generator=torch.Generator().manual_seed(seed))


def _box(b=1, box=(100, 300, 60, 333), dtype=torch.bool):
    return CP.box_mask(b, 512, box, dtype)


def _batch2(req, seed):
    """The request on a batch-2 latent."""
    x = torch.randn((2, 4, 64, 64), generator=torch.Generator().manual_seed(seed))
    return replace(req, input=dict(req.input, x=x))


def _inpaint(req, seed, strength=1.0, mask=None, b_init=1):
    return replace(req, x_init=_x_init(500 + seed, b_init), strength=strength, seed=seed,
                   repaint_mask=_box() if mask is None else mask)


def _shape(req):
    inp = req.input[0] if isinstance(req.input, list) else req.input
    return tuple(inp["x"].shape)


@contextmanager
def _seeded_q_sample(diffusion, seed):
    diffusion.q_sample = CP.seeded_q_sample(diffusion, seed)
    try:
        yield
    finally:
        del diffusion.q_sample


def _alone(diffusion, req, model=None):
    """The request through its own sampler kind on a fresh fake: `_sample` (what every sampler's `sample` calls, and
    `sample_loop(mis=)` for a Multi-instance request) with mask = the keep mask, x0 = x_init over the batch and
    `diffusion.q_sample` drawing the seeded blend noise."""
    model = FakeUNet() if model is None else model
    req = _fresh(req)
    kw = dict(alpha_generator_func=req.alpha_generator_func, set_alpha_scale=set_alpha_scale)
    multi = isinstance(req.input, list)
    shape = _shape(req)
    kind = {"ddim": DDIMSampler, "dpmpp_2m": DPMSolverSampler}.get(req.sampler, PLMSSamplerInst if multi else PLMSSampler)
    s = kind(diffusion, model, **kw)
    mask = x0 = None
    if req.repaint_mask is not None:
        mask = CP.keep_of(req.repaint_mask).float()[:, None]
        x0 = req.x_init.expand(shape)
    with _seeded_q_sample(diffusion, req.seed):
        return s._sample(req.S, shape, req.input, req.uc, req.guidance_scale, mask, x0, req.x_init, req.strength,
                         req.seed, eta=req.eta, mis=req.mis if multi else None)


def _engine(diffusion, reqs, arrivals=None, **kw):
    """The requests through a SamplingEngine, request j submitted before tick arrivals[j]."""
    eng = SamplingEngine(FakeUNet(), diffusion, max_batch=8, **kw)
    arrivals = arrivals or [0] * len(reqs)
    tickets, done, tick = {}, {}, 0
    while len(done) < len(reqs):
        for j, r in enumerate(reqs):
            if arrivals[j] == tick:
                tickets[eng.submit(_fresh(r))] = j
        done.update({tickets[t]: v for t, v in eng.step().items()})
        tick += 1
    return [done[j] for j in range(len(reqs))]


# ------------------------------------------------------------------------------------------------
# validation and the mask reduction
# ------------------------------------------------------------------------------------------------
def test_check_requests_repaint_mask():
    ok = _req(1, S)
    plans = check_requests([_inpaint(ok, 3), _inpaint(ok, 4, strength=0.35, mask=_box(dtype=torch.uint8))], S, 32)
    assert [p.k0 for p in plans] == [0, 7]
    check_requests([replace(ok, init_image=CE.random_images(1, 512, 512, 1), repaint_mask=_box(), seed=1)], S, 32)
    b2 = _batch2(ok, 5)
    check_requests([_inpaint(b2, 5, mask=_box(2)), _inpaint(b2, 6, b_init=2)], S, 32)
    bad = [
        (_box().float(), "repaint_mask must be a bool or uint8 tensor"),
        (_box().to(torch.int32), "repaint_mask must be a bool or uint8 tensor"),
        (_box()[0], "does not fit the latent"),  # rank 2
        (_box()[:, :256], "does not fit the latent"),  # not 8x the latent
        (_box(2), "does not fit the latent"),  # batch 2 on a batch-1 request
        (_box()[..., None], "does not fit the latent"),
    ]
    for m, msg in bad:
        with pytest.raises(ValueError, match=f"request 1: (repaint_mask of shape .* )?{msg}"):
            check_requests([ok, _inpaint(ok, 2, mask=m)], S, 32)
    with pytest.raises(ValueError, match="request 1: repaint_mask needs x_init or init_image"):
        check_requests([ok, replace(ok, repaint_mask=_box())], S, 32)
    with pytest.raises(ValueError, match="inpainting.*use repaint_mask with x_init or init_image"):
        check_requests([replace(_inpaint(ok, 2), mask=torch.zeros((1, 4, 64, 64)), x0=torch.zeros((1, 4, 64, 64)))],
                       S, 32)
    with pytest.raises(ValueError, match="inpainting"):
        check_requests([replace(_inpaint(ok, 2), x0=torch.zeros((1, 4, 64, 64)))], S, 32)


def test_engine_submit_validates(diffusion):
    eng = SamplingEngine(FakeUNet(), diffusion)
    with pytest.raises(ValueError, match="repaint_mask needs x_init or init_image"):
        eng.submit(replace(_req(1, S), repaint_mask=_box()))
    with pytest.raises(ValueError, match="repaint_mask must be a bool or uint8 tensor"):
        eng.submit(_inpaint(_req(1, S), 2, mask=_box().float()))
    assert eng.queued == []


def test_keep_mask_reduction():
    g = torch.Generator().manual_seed(0)
    m = (torch.rand((3, 64, 48), generator=g) < 0.01).to(torch.uint8) * 7  # sparse: some cells keep, some repaint
    keep = keep_mask(m)
    assert keep.dtype == torch.uint8 and keep.shape == (3, 8, 6)
    assert torch.equal(keep, CP.keep_of(m)) and torch.equal(keep, keep_mask(m.bool()))
    for b, y, x in [(0, 0, 0), (1, 3, 4), (2, 7, 5)]:
        assert keep[b, y, x] == int(not m[b, 8 * y:8 * y + 8, 8 * x:8 * x + 8].any())
    box = keep_mask(_box(box=(8, 17, 0, 8)))  # rows 8..16: latent rows 1 and 2 (one pixel of row 2)
    assert box[0, :, 0].tolist() == [1, 0, 0, 1, 1, 1, 1, 1] + [1] * 56 and int(box[0, :, 1:].sum()) == 64 * 63


# ------------------------------------------------------------------------------------------------
# the drivers against each request's own sampler
# ------------------------------------------------------------------------------------------------
def _targets():
    """Inpainting requests of every sampler kind: PLMS at strength 1 and 0.6, DDIM at eta 0 and (batch 2, batch-1
    source and mask) eta 0.7, DPM-Solver++ at 0.8, Multi-instance PLMS at strength 1 (merges at step 3)."""
    return [
        _inpaint(_req(11, S), 21),
        _inpaint(_req(12, S), 22, strength=0.6, mask=_box(dtype=torch.uint8)),
        _inpaint(_req(13, S, sampler="ddim"), 23),
        _inpaint(_batch2(_req(14, S, sampler="ddim", eta=0.7), 14), 24, strength=0.9),
        _inpaint(_req(15, S, sampler="dpmpp_2m"), 25, strength=0.8, mask=_box(box=(0, 512, 256, 512))),
        _inpaint(_req(16, S, n=2, mis=0.36), 26),
    ]


def _neighbours():
    """A plain PLMS request and an image-to-image DDIM request."""
    return [_req(31, S), replace(_req(32, S, sampler="ddim", eta=0.5), x_init=_x_init(9), strength=0.6, seed=9)]


@pytest.mark.parametrize("k", range(6))
def test_sample_requests_match_each_request_alone(diffusion, torch_kernels, k):
    target = _targets()[k]
    reqs = [_neighbours()[0], target, _neighbours()[1]]
    want = _alone(diffusion, target)
    got = sample_requests(FakeUNet(), diffusion, [_fresh(r) for r in reqs], S, max_batch=8)
    assert torch.equal(got[1], want)
    assert torch.equal(got[0], _alone(diffusion, reqs[0])) and torch.equal(got[2], _alone(diffusion, reqs[2]))
    # the blend keeps the source: a run without the mask differs
    assert not torch.allclose(want, _alone(diffusion, replace(target, repaint_mask=None)), rtol=1e-3, atol=1e-4)


@pytest.mark.parametrize("k", range(6))
def test_engine_matches_each_request_alone(diffusion, torch_kernels, k):
    target = _targets()[k]
    reqs = [_neighbours()[0], target, _neighbours()[1], replace(_req(33, S + 1), S=S + 1)]
    got = _engine(diffusion, reqs, [0, 1, 1, 3])
    assert torch.equal(got[1], _alone(diffusion, target))
    assert torch.equal(got[3], _alone(diffusion, reqs[3]))


# ------------------------------------------------------------------------------------------------
# edges
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [0, 3, 5])
def test_all_repaint_is_the_request_without_mask(diffusion, torch_kernels, k):
    target = _targets()[k]
    full = replace(target, repaint_mask=torch.ones((1, 512, 512), dtype=torch.uint8))
    plain = replace(target, repaint_mask=None)
    got = sample_requests(FakeUNet(), diffusion, [_fresh(full), _fresh(plain)], S, max_batch=8)
    assert torch.equal(got[0], got[1])
    assert torch.equal(_engine(diffusion, [full])[0], got[1])


class RecordingUNet(FakeUNet):
    """FakeUNet that logs (timestep, latent) of every input."""

    def __init__(self):
        super().__init__()
        self.seen = []

    def forward_batched(self, inputs, *, scales=None, restored=None):
        self.seen += [(int(i["timesteps"].reshape(-1)[0]), i["x"].clone()) for i in inputs]
        return super().forward_batched(inputs, scales=scales, restored=restored)


@pytest.mark.parametrize("sampler", ["plms", "ddim"])
def test_all_keep_blends_every_evaluation_but_the_corrector(diffusion, torch_kernels, sampler):
    """With every cell kept, the latent of every evaluation is q_sample(x_init, t) with the seeded noise, except the
    corrector's evaluation of the first PLMS step, which takes the predictor's latent at t_next unblended."""
    req = replace(_inpaint(_req(41, S, sampler=sampler), 41, strength=0.6,
                           mask=torch.zeros((1, 512, 512), dtype=torch.bool)), uc=None)
    for drive in ("sample_requests", "engine"):
        model = RecordingUNet()
        if drive == "sample_requests":
            sample_requests(model, diffusion, [_fresh(req)], S, max_batch=8)
        else:
            eng = SamplingEngine(model, diffusion, max_batch=8, buckets=None)  # no padding inputs
            eng.submit(_fresh(req))
            eng.drain()
        ts = [t for t, _ in model.seen]
        steps = np.flip(np.asarray(list(range(0, 1000, 1000 // S))) + 1)
        steps = steps[CI.start_step(len(steps), 0.6):]
        want_ts = list(steps)
        if sampler == "plms":
            want_ts.insert(1, steps[1])  # the corrector's evaluation at t_next of the first step
        assert ts == [int(t) for t in want_ts], (ts, want_ts)
        for j, (t, x) in enumerate(model.seen):
            q = CP.q_value(req.x_init, float(diffusion.sqrt_alphas_cumprod[t]),
                           float(diffusion.sqrt_one_minus_alphas_cumprod[t]), req.seed, t, x.shape)
            assert torch.equal(x, q) != (sampler == "plms" and j == 1), (drive, j, t)


# ------------------------------------------------------------------------------------------------
# image outputs
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("b", [1, 2])
def test_paste_back(diffusion, torch_kernels, b):
    """An init_image request with a box mask and output="image": the bytes outside the mask are the source's, the ones
    inside it the decode of the request's latent; a request from x_init gets the decode as it is."""
    src = CE.random_images(1, 512, 512, 77)
    base = _req(51, S) if b == 1 else _batch2(_req(51, S), 51)
    req = replace(base, init_image=src, repaint_mask=_box(b), seed=5, output="image")
    lat = replace(req, output="latent")
    from_latent = replace(_inpaint(base, 6, mask=_box(1)), output="image")
    vae = CE.FakeAutoencoder()
    for got in (sample_requests(FakeUNet(), diffusion, [_fresh(r) for r in (req, lat, from_latent)], S,
                                autoencoder=vae),
                _engine(diffusion, [req, lat, from_latent], autoencoder=vae)):
        img, z = got[0], got[1]
        assert img.dtype == torch.uint8 and img.shape == (b, 512, 512, 3)
        dec = vae.decode_images(z)
        rep = _box(b)[..., None].expand(b, 512, 512, 3)
        assert torch.equal(img[~rep], src.expand(b, -1, -1, -1)[~rep])
        assert torch.equal(img[rep], dec[rep])
        assert not torch.equal(dec[~rep], img[~rep])  # the decode alone does not keep the bytes
        assert torch.equal(got[2], vae.decode_images(_alone(diffusion, from_latent)))
