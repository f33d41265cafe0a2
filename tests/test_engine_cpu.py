"""Host logic of the continuous-batching engine (instancediffusion_b200.ldm.models.diffusion.engine): admission, the
tick in which each evaluation, merge and finish happens, bucket padding, grouping by latent size, and the validation
of `submit`.  Driven by the fake model of fake_unet.py, so no GPU is needed; each request's latent is compared with its
own sampler run on the same fake."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from fake_unet import FakeUNet, _alone, _fresh, _req, torch_kernels  # noqa: E402,F401
from instancediffusion_b200.ldm.models.diffusion.batched import RequestPlan, schedule_steps  # noqa: E402
from instancediffusion_b200.ldm.models.diffusion.engine import SamplingEngine, pick_bucket, plan_forwards  # noqa: E402

pytestmark = pytest.mark.usefixtures("torch_kernels")


@pytest.fixture
def diffusion():
    from instancediffusion_b200.ldm.models.diffusion.ldm import LatentDiffusion
    return LatentDiffusion(linear_start=0.00085, linear_end=0.012, timesteps=1000)


def _run(engine, arrivals):
    """arrivals: {tick: [request]} -> ({ticket: tick it finished in}, {ticket: latent}, {ticket: request})."""
    finished, out, reqs, tick = {}, {}, {}, 0
    while tick <= max(arrivals) or engine.queued or engine.live:
        for r in arrivals.get(tick, []):
            reqs[engine.submit(_fresh(r))] = r
        for t, x in engine.step().items():
            finished[t], out[t] = tick, x
        tick += 1
    return finished, out, reqs


@pytest.mark.parametrize("S,steps", [(10, 10), (11, 12), (20, 20)])
def test_finishing_tick_and_corrector_tick(diffusion, S, steps):
    """A request admitted at tick a evaluates step 0 at a, its corrector at a + 1, and finishes at a + steps."""
    model = FakeUNet()
    eng = SamplingEngine(model, diffusion, buckets=None)
    req = _req(1, S)
    finished, out, _ = _run(eng, {2: [req]})
    assert finished == {0: 2 + steps}
    ts = [c["t"][0] for c in model.calls]
    assert len(ts) == steps + 1 and ts[0] > ts[1]
    assert ts[1] == ts[2]  # the corrector evaluates at t_next, the tick after the predictor; step 1 at the same t
    assert torch.allclose(out[0], _alone(diffusion, req), rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("mis,S,merge_tick", [(0.36, 10, 4), (0.36, 11, 5), (1.0, 10, 11)])
def test_merge_tick(diffusion, mis, S, merge_tick):
    """A 2-instance request (3 trajectories x cond/uncond) evaluates 6 images per tick until its merge, then 2: the
    merge before step int(steps * mis) lands in tick merge_step + 1 (the corrector tick comes first); mis = 1 merges
    after the last step, in the finishing tick."""
    model = FakeUNet()
    eng = SamplingEngine(model, diffusion, buckets=None)
    req = _req(2, S, n=2, mis=mis)
    finished, out, _ = _run(eng, {0: [req]})
    per_tick = [sum(c["sizes"]) for c in model.calls]
    assert len(per_tick) == schedule_steps(S) + 1 and finished == {0: schedule_steps(S)}
    assert per_tick == [6] * merge_tick + [2] * (len(per_tick) - merge_tick)
    assert torch.allclose(out[0], _alone(diffusion, req), rtol=1e-5, atol=1e-6)


def test_fifo_admission_under_max_live_images(diffusion):
    model = FakeUNet()
    eng = SamplingEngine(model, diffusion, max_batch=8, max_live_images=8, buckets=None)
    big, small = _req(3, 10, n=2, mis=0.36), _req(4, 10)   # 6 and 2 images
    tickets = [eng.submit(_fresh(r)) for r in (big, big, small)]
    assert eng.queued == tickets and eng.live == []
    eng.step()
    assert eng.live == [0] and eng.queued == [1, 2]  # 6 + 6 > 8; the small request waits behind it (FIFO)
    done = {}
    while eng.queued or eng.live:
        done.update(eng.step())
        assert sum(6 if t < 2 else 2 for t in eng.live) <= 8
    assert set(done) == set(tickets)
    for t, r in zip(tickets, (big, big, small)):
        assert torch.allclose(done[t], _alone(diffusion, r), rtol=1e-5, atol=1e-6)
    # finished requests' hoisted entries are dropped, except those a queued or live request shares (the second request
    # is a copy of the first with the same context tensors)
    first, last = model.dropped[0], model.dropped[-1]
    assert set(first[0]) <= set(first[1]) and last[1] == []


def test_staggered_requests_match_their_own_samplers(diffusion):
    model = FakeUNet()
    eng = SamplingEngine(model, diffusion, max_batch=8)
    arrivals = {0: [_req(5, 10, n=2, mis=0.36), _req(6, 11, n=1, mis=1.0)], 3: [_req(7, 20)], 7: [_req(8, 11, n=3, mis=0.36)],
                12: [_req(9, 10, alpha=None)]}
    _, out, reqs = _run(eng, arrivals)
    for t, r in reqs.items():
        assert torch.allclose(out[t], _alone(diffusion, r), rtol=1e-5, atol=1e-6), t
    assert all(sum(c["sizes"]) in (2, 4, 8, 16, 24, 32) for c in model.calls)


def test_bucket_choice_and_padding_rows(diffusion):
    assert [pick_bucket(n, 1, (2, 4, 8)) for n in (1, 2, 3, 5, 8, 9)] == [2, 2, 4, 8, 8, None]
    assert pick_bucket(6, 2, (2, 4, 8)) == 8 and pick_bucket(5, 2, (8, 9)) == 9 and pick_bucket(3, 1, None) is None
    model = FakeUNet()
    eng = SamplingEngine(model, diffusion, max_batch=4, buckets=(4, 8))
    eng.submit(_req(10, 10, n=1, mis=0.36))  # 4 images
    eng.submit(_req(11, 10))                  # 2 images
    eng.step()
    (c1, c2) = model.calls
    assert c1["sizes"] == [1] * 4 and c2["sizes"] == [1] * 2 + [1] * 2  # 4 | 2 padded to 4
    assert c2["zero"] == [False, False, True, True] and c2["scales"][2:] == [0.0, 0.0]
    assert c2["restored"][2:] == [False, False] and c2["t"][2:] == c2["t"][1:2] * 2
    assert eng.padded_images == 2 and eng.forwards == 2


def test_latent_sizes_run_in_separate_forwards(diffusion):
    model = FakeUNet()
    eng = SamplingEngine(model, diffusion, max_batch=32, buckets=None)
    a, b, c = _req(12, 10), _req(13, 10, size=48), _req(14, 10, ctx=64)
    _, out, reqs = _run(eng, {0: [a, b, c]})
    assert [set(cl["hw"]) for cl in model.calls[:3]] == [{(64, 64)}, {(48, 48)}, {(64, 64)}]
    for t, r in reqs.items():
        assert torch.allclose(out[t], _alone(diffusion, r), rtol=1e-5, atol=1e-6)
    slots = [(0, 0), (1, 0), (2, 0), (3, 0)]
    plans = [RequestPlan(1, None, 1, True)] * 4
    fw = plan_forwards(slots, plans, ["a", "b", "a", "b"], 32, (2, 4))
    assert fw == [([(0, 0), (2, 0)], 4), ([(1, 0), (3, 0)], 4)]


def test_submit_validation(diffusion):
    model = FakeUNet()
    eng = SamplingEngine(model, diffusion, max_batch=4, max_live_images=8)
    with pytest.raises(ValueError, match="S"):
        eng.submit(_req(20, None))
    with pytest.raises(ValueError, match="S must be"):
        eng.submit(_req(20, 0))
    with pytest.raises(ValueError, match="S must be"):
        eng.submit(_req(20, 1001))
    with pytest.raises(ValueError, match="input list"):
        eng.submit(_req(20, 10, mis=0.36))
    with pytest.raises(ValueError, match="outside"):
        eng.submit(_req(20, 10, n=2, mis=1.5))
    with pytest.raises(ValueError, match="inpainting"):
        eng.submit(_req(20, 10, mask=torch.zeros((1, 4, 64, 64)), x0=torch.zeros((1, 4, 64, 64))))
    with pytest.raises(ValueError, match="max_live_images"):
        eng.submit(_req(20, 10, n=4, mis=0.36))  # 5 trajectories x 2 images
    assert eng.queued == []
    uneven = FakeUNet()
    uneven.fusers[1].scale = 0.25
    with pytest.raises(ValueError, match="differs between fusers"):
        SamplingEngine(uneven, diffusion).submit(_req(20, 10, alpha=None))
    SamplingEngine(uneven, diffusion).submit(_req(20, 10))  # a request with an alpha schedule sets its own scale
    with pytest.raises(ValueError, match="max_batch"):
        SamplingEngine(model, diffusion, max_batch=0)
