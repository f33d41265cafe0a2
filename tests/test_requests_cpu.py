"""Host logic of the batched request sampler (instancediffusion_b200.ldm.models.diffusion.batched): the step planner
that builds each step's forward chunks, the validation of a request list, and whole `sample_requests` runs on the fake
model of fake_unet.py.  No GPU needed."""
import os
import sys
from functools import partial

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from fake_unet import AGEN, FakeUNet, _alone, _fresh, _latent_mean, _plms_update, _req  # noqa: E402
from instancediffusion_b200 import ops  # noqa: E402
from instancediffusion_b200.ldm.models.diffusion.batched import (  # noqa: E402
    Request, RequestPlan, check_requests, plan_chunks, plan_step, sample_requests, schedule_steps)
from instancediffusion_b200.ldm.modules.diffusionmodules.util import make_ddim_timesteps  # noqa: E402
from instancediffusion_b200.utils.model import alpha_generator  # noqa: E402


def _inp(b=1, size=64, ctx=77):
    return dict(x=torch.zeros((b, 4, size, size)), timesteps=None, context=torch.zeros((b, ctx, 768)))


def _mis_request(n, b=1, mis=0.36, **kw):
    return Request(input=[_inp(b) for _ in range(n + 1)], uc=torch.zeros((b, 77, 768)), guidance_scale=7.5, mis=mis, **kw)


def test_plans_of_plain_and_mis_requests():
    reqs = [Request(input=_inp(), uc=torch.zeros((1, 77, 768)), guidance_scale=7.5),
            _mis_request(3, b=2),
            Request(input=_inp(), uc=None),                                       # no CFG: one row per image
            Request(input=_inp(), uc=torch.zeros((1, 77, 768)), guidance_scale=1.0)]  # gs 1: no uncond rows
    plans = check_requests(reqs, 50, 32)
    assert plans[0] == RequestPlan(1, None, 1, True)
    assert plans[1] == RequestPlan(4, 18, 2, True)  # int(50 * 0.36) = 18
    assert not plans[2].cfg and not plans[3].cfg
    assert plans[1].rows() == 4 and plans[2].rows() == 1


def test_trajectory_counts_and_merge_steps():
    p = RequestPlan(trajectories=4, merge_step=3, images=1, cfg=True)
    assert [p.live(i) for i in range(6)] == [4, 4, 4, 1, 1, 1]
    assert [RequestPlan(1, None, 1, True).live(i) for i in range(3)] == [1, 1, 1]
    # mis = 0 with an input list merges before the first step
    assert RequestPlan(3, 0, 1, True).live(0) == 1
    plans = [RequestPlan(1, None, 1, True), RequestPlan(4, 3, 1, True), RequestPlan(6, 5, 1, True)]
    for i, want in [(0, 11), (2, 11), (3, 8), (4, 8), (5, 3), (9, 3)]:
        slots = [s for c in plan_step(plans, i, 1000) for s in c]
        assert len(slots) == want, (i, slots)
        assert len(set(slots)) == len(slots)


def test_merge_step_follows_the_schedule_length():
    """The PLMS schedule of S steps is range(0, 1000, 1000 // S): 31 steps for S = 30, 12 for S = 11.  The merge comes
    before step int(len * mis), as PLMSSamplerInst computes it, and mis = 1 merges after the last step."""
    assert [schedule_steps(S) for S in (10, 11, 30, 50, 60)] == [10, 12, 31, 50, 63]
    assert check_requests([_mis_request(2)], 30, 32)[0].merge_step == 11   # not int(30 * 0.36) = 10
    assert check_requests([_mis_request(2)], 11, 32)[0].merge_step == 4    # not 3
    assert check_requests([_mis_request(2, mis=1.0)], 30, 32)[0].merge_step == 31
    plans = check_requests([_mis_request(2, mis=1.0)], 11, 32)
    assert [plans[0].live(i) for i in range(12)] == [3] * 12
    with pytest.raises(ValueError, match="S must be"):
        check_requests([_mis_request(2)], 1001, 32)


def test_max_batch_chunking_keeps_trajectories_whole():
    plans = [RequestPlan(1, None, 1, True), RequestPlan(5, 2, 2, True), RequestPlan(1, None, 3, False)]
    chunks = plan_step(plans, 0, 8)
    # rows: req0 -> 2, req1 -> 5 trajectories x 4, req2 -> 3
    sizes = [sum(plans[r].rows() for r, _ in c) for c in chunks]
    assert sizes == [6, 8, 8, 3] and all(s <= 8 for s in sizes)
    assert [s for c in chunks for s in c] == [(0, 0), (1, 0), (1, 1), (1, 2), (1, 3), (1, 4), (2, 0)]
    # a trajectory larger than max_batch gets a chunk of its own
    big = [RequestPlan(1, None, 4, True), RequestPlan(1, None, 1, True)]
    assert plan_chunks([(0, 0), (1, 0)], big, 4) == [[(0, 0)], [(1, 0)]]
    # after the merge the MIS request contributes one trajectory
    assert sum(len(c) for c in plan_step(plans, 2, 8)) == 3


def test_validation_errors():
    ok = Request(input=_inp(), uc=torch.zeros((1, 77, 768)), guidance_scale=7.5)
    with pytest.raises(ValueError, match="S="):
        check_requests([ok, Request(input=_inp(), S=20)], 10, 32)
    with pytest.raises(ValueError, match="latent"):
        check_requests([ok, Request(input=_inp(size=48))], 10, 32)
    with pytest.raises(ValueError, match="context length"):
        check_requests([ok, Request(input=_inp(ctx=64))], 10, 32)
    with pytest.raises(ValueError, match="context length"):
        check_requests([Request(input=_inp(), uc=torch.zeros((1, 64, 768)), guidance_scale=7.5)], 10, 32)
    with pytest.raises(ValueError, match="inpainting"):
        check_requests([Request(input=_inp(), mask=torch.zeros((1, 4, 64, 64)), x0=torch.zeros((1, 4, 64, 64)))], 10, 32)
    with pytest.raises(ValueError, match="input list"):
        check_requests([Request(input=_inp(), mis=0.36)], 10, 32)
    with pytest.raises(ValueError, match="latent shapes"):
        check_requests([Request(input=[_inp(1), _inp(2)], mis=0.36)], 10, 32)
    with pytest.raises(ValueError, match="max_batch"):
        check_requests([ok], 10, 0)
    with pytest.raises(ValueError, match="no requests"):
        check_requests([], 10, 32)
    # a request without x gives its latent shape explicitly
    plans = check_requests([Request(input=dict(x=None, timesteps=None, context=torch.zeros((2, 77, 768))),
                                    shape=(2, 4, 64, 64))], 10, 32)
    assert plans[0].images == 2


@pytest.mark.parametrize("S", [10, 11])
def test_sample_requests_forwards_and_latents(monkeypatch, S):
    """Plain, mis 0.36, mis 1.0 and no-alpha-schedule requests in one run on the fake UNet, its fusers at 0.5: every
    forward (images, timesteps, fuser scales and conv flags per input, the corrector forwards of step 0 after the
    predictor's), the model's conv and fuser scale afterwards, and each latent against the request's own sampler."""
    from instancediffusion_b200.ldm.models.diffusion.ldm import LatentDiffusion
    monkeypatch.setattr(ops, "plms_update", _plms_update)
    monkeypatch.setattr(ops, "latent_mean", _latent_mean)
    diffusion = LatentDiffusion(linear_start=0.00085, linear_end=0.012, timesteps=1000)
    ones = partial(alpha_generator, type=[1.0, 0.0, 0.0])
    reqs = [_req(31, S), _req(32, S, n=2, mis=0.36), _req(33, S, n=1, mis=1.0, alpha=ones), _req(34, S, alpha=None)]
    model = FakeUNet(scale=0.5)
    got = sample_requests(model, diffusion, [_fresh(r) for r in reqs], S, max_batch=8)
    # a sequential run leaves the SD1.5 conv of the first two requests and the last alpha of the last alpha schedule
    assert model._first_conv_restored and [f.scale for f in model.fusers] == [1.0, 1.0]

    steps = schedule_steps(S)
    t = [int(v) for v in np.flip(make_ddim_timesteps("uniform", S, 1000))]
    alphas = [AGEN(steps), AGEN(steps), ones(steps), None]
    plans = check_requests(reqs, S, 8)
    want = []
    for i in range(steps):
        scale = [0.5 if a is None else float(a[i]) for a in alphas]
        sd_conv = [a is not None and 0 in a[:i + 1] for a in alphas]  # from a request's first alpha-0 step on
        for ts in ([t[0], t[1]] if i == 0 else [t[i]]):
            for chunk in plan_step(plans, i, 8):
                rows = [r for r, _ in chunk for _ in ("cond", "uncond")]
                want.append(dict(sizes=[1] * len(rows), t=[ts] * len(rows), scales=[scale[r] for r in rows],
                                 restored=[sd_conv[r] for r in rows]))
    assert [{k: c[k] for k in want[0]} for c in model.calls] == want
    for k, r in enumerate(reqs):
        assert torch.allclose(got[k], _alone(diffusion, r, scale=0.5), rtol=1e-5, atol=1e-6), k

    model = FakeUNet(scale=0.5)
    model.fusers[1].scale = 0.25
    with pytest.raises(ValueError, match="differs between fusers"):
        sample_requests(model, diffusion, [_fresh(r) for r in reqs], S)
