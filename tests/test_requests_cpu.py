"""Host logic of the batched request sampler (instancediffusion_b200.ldm.models.diffusion.batched): the step planner
that builds each step's forward chunks, and the validation of a request list.  No GPU needed."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from instancediffusion_b200.ldm.models.diffusion.batched import (  # noqa: E402
    Request, RequestPlan, check_requests, plan_chunks, plan_step)


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
    from instancediffusion_b200.ldm.models.diffusion.batched import schedule_steps
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
