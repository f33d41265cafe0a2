"""DDIM sampling without a GPU: `DDIMSampler.make_schedule` against a float64 restatement of util.py:73-83, the torch
restatement of the reference's DDIM loop against its latents (tests/golden/ddim.pt), the drop-in path, request
validation, and DDIM requests mixed with PLMS ones in `sample_requests` / `SamplingEngine` on the fake UNet of
fake_unet.py (the kernel replaced by its torch restatement with the mirrored noise; the noise stream itself is tested
in test_noise_streams_cpu.py)."""
import os
import subprocess
import sys
from dataclasses import replace

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import cases  # noqa: E402
import cases_ddim as CD  # noqa: E402
from fake_unet import AGEN, FakeUNet, _alone, _fresh, _req, torch_kernels  # noqa: E402,F401
from instancediffusion_b200.ldm.models.diffusion.batched import (  # noqa: E402
    Request, RequestPlan, _RequestState, check_requests, sample_requests, schedule_steps)
from instancediffusion_b200.ldm.models.diffusion.ddim import DDIMSampler  # noqa: E402
from instancediffusion_b200.ldm.models.diffusion.engine import SamplingEngine  # noqa: E402
from instancediffusion_b200.utils.model import set_alpha_scale  # noqa: E402

GOLDEN = os.path.join(HERE, "golden")
ROOT = os.path.dirname(HERE)


@pytest.fixture
def diffusion():
    from instancediffusion_b200.ldm.models.diffusion.ldm import LatentDiffusion
    return LatentDiffusion(linear_start=0.00085, linear_end=0.012, timesteps=1000)


# ------------------------------------------------------------------------------------------------
# schedule and the reference restatement
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S", [4, 10, 30, 50])
@pytest.mark.parametrize("eta", [0.0, 0.5, 1.0])
def test_schedule_matches_float64_restatement(diffusion, S, eta):
    s = DDIMSampler(diffusion, FakeUNet())
    s.make_schedule(S, ddim_eta=eta)
    steps, a, a_prev, sig = CD.ddim_schedule(S, eta, diffusion.alphas_cumprod)
    assert len(s.ddim_timesteps) == len(steps) == schedule_steps(S)
    assert np.array_equal(s.ddim_timesteps, steps)
    assert np.array_equal(s.ddim_alphas.double().numpy(), a)
    assert np.array_equal(np.asarray(s.ddim_alphas_prev, dtype=np.float64), a_prev)
    np.testing.assert_allclose(np.asarray(s.ddim_sigmas, dtype=np.float64), sig, rtol=1e-12, atol=0)
    assert (1 - a_prev - sig ** 2 >= -1e-12).all()  # the direction term's radicand at eta <= 1
    if S == 30:
        assert len(steps) == 31


def test_plms_schedule_still_rejects_eta(diffusion):
    from instancediffusion_b200.ldm.models.diffusion.plms import PLMSSampler
    with pytest.raises(ValueError, match="eta"):
        PLMSSampler(diffusion, FakeUNet()).make_schedule(10, ddim_eta=0.5)
    with pytest.raises(ValueError, match="eta"):
        DDIMSampler(diffusion, FakeUNet()).make_schedule(10, ddim_eta=-0.1)


def _load(name):
    path = os.path.join(GOLDEN, name)
    if not os.path.exists(path):
        pytest.skip(f"{name} not generated")
    return torch.load(path, map_location="cpu")


@pytest.fixture(scope="module")
def unet_sd():
    import json
    from instancediffusion_b200.weights import synth_tensor
    path = os.path.join(GOLDEN, "unet_schema.json")
    if not os.path.exists(path):
        pytest.skip("unet_schema.json not generated")
    schema = json.load(open(path))
    return {k: synth_tensor(k, tuple(s), cases.UNET_CASE["weight_seed"]) for k, s in schema.items()}


@pytest.mark.parametrize("name", list(CD.DDIM_CASES))
def test_ddim_sample_restatement_matches_reference(unet_sd, name):
    """cases_ddim.ddim_sample vs the latents of the reference's DDIMSampler (tests/golden/ddim.pt), fp32 vs fp32."""
    from oracle import torch_oracle as TO
    from instancediffusion_b200.grounding_input.text_grounding_tokinzer_input import GroundingNetInput
    from instancediffusion_b200.weights import UNIFUSION_FLAGS
    gold = _load("ddim.pt")
    sc = CD.DDIM_CASES[name]
    sd15 = _load("sd15_first_conv.pt")
    flags = UNIFUSION_FLAGS["box"]
    inp, uc = CD.ref_inputs_for(GroundingNetInput(), name)
    null_gi = TO.null_grounding_input(inp["grounding_input"])

    def eval_fn(i, alpha):
        gi = i.get("grounding_input")
        return TO.unet_forward(unet_sd, i["x"], i["timesteps"], i["context"], gi if gi is not None else null_gi,
                               flags, scale=float(alpha), first_conv=sd15 if alpha == 0 else None)

    with torch.no_grad():
        x = CD.ddim_sample(eval_fn, inp, uc, sc["S"], sc["guidance"], alpha_type=sc["alpha_type"])
    rel = ((x - gold[name]).norm() / gold[name].norm()).item()
    print(f"[ddim_sample restatement] {name}: rel_l2 {rel:.2e}")
    assert rel < 2e-4, rel


# ------------------------------------------------------------------------------------------------
# drop-in path and validation
# ------------------------------------------------------------------------------------------------
def test_dropin_resolves_ddim_to_the_mirror():
    code = (
        "import sys; sys.path.insert(0, %r)\n"
        "from instancediffusion_b200 import dropin; dropin.install()\n"
        "from ldm.models.diffusion.ddim import DDIMSampler\n"
        "import instancediffusion_b200.ldm.models.diffusion.ddim as M\n"
        "assert DDIMSampler is M.DDIMSampler, DDIMSampler.__module__\n"
        "print('ok')\n" % ROOT)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "ok" in r.stdout, r.stderr[-2000:]


def _inp(b=1, size=64, ctx=77):
    return dict(x=torch.zeros((b, 4, size, size)), timesteps=None, context=torch.zeros((b, ctx, 768)))


def test_request_validation():
    uc = torch.zeros((1, 77, 768))
    ok = Request(input=_inp(), uc=uc, guidance_scale=7.5)
    assert ok.sampler == "plms" and ok.eta == 0.0 and ok.seed is None
    assert check_requests([ok], 10, 32) == [RequestPlan(1, None, 1, True)]
    ddim = Request(input=_inp(2), uc=torch.zeros((2, 77, 768)), guidance_scale=7.5, sampler="ddim", eta=0.5, seed=3)
    assert check_requests([ok, ddim], 10, 32) == [RequestPlan(1, None, 1, True), RequestPlan(1, None, 2, True)]
    with pytest.raises(ValueError, match="unknown sampler"):
        check_requests([replace(ok, sampler="dpm")], 10, 32)
    with pytest.raises(ValueError, match="eta"):
        check_requests([replace(ddim, eta=-0.5)], 10, 32)
    with pytest.raises(ValueError, match="eta"):
        check_requests([replace(ddim, eta=float("nan"))], 10, 32)
    with pytest.raises(ValueError, match="sampler='ddim'"):
        check_requests([replace(ok, eta=0.5)], 10, 32)
    with pytest.raises(ValueError, match="PLMS only"):
        check_requests([Request(input=[_inp(), _inp()], uc=uc, guidance_scale=7.5, mis=0.36, sampler="ddim")], 10, 32)
    with pytest.raises(ValueError, match="PLMS only"):
        check_requests([Request(input=[_inp(), _inp()], uc=uc, guidance_scale=7.5, sampler="ddim")], 10, 32)
    with pytest.raises(ValueError, match="PLMS only"):
        check_requests([replace(ddim, mis=0.36)], 10, 32)
    with pytest.raises(ValueError, match="seed"):
        check_requests([replace(ddim, seed=-1)], 10, 32)
    with pytest.raises(ValueError, match="inpainting"):  # still rejected for DDIM requests
        check_requests([replace(ddim, mask=torch.zeros((2, 4, 64, 64)), x0=torch.zeros((2, 4, 64, 64)))], 10, 32)


def test_ddim_sampler_rejects_an_input_list(diffusion):
    with pytest.raises(ValueError, match="input dict"):
        DDIMSampler(diffusion, FakeUNet()).sample(10, (1, 4, 64, 64), [_inp(), _inp()])


def test_unseeded_requests_draw_from_torchs_generator_in_order(diffusion):
    reqs = [replace(_req(k, 10), sampler="ddim", eta=0.5) for k in (1, 2)]
    torch.manual_seed(99)
    want = [int(torch.randint(0, 2 ** 63 - 1, (1,), dtype=torch.int64).item()) for _ in reqs]
    model = FakeUNet()  # its fusers' initialisation draws from the generator too
    torch.manual_seed(99)
    plans = check_requests(reqs, 10, 32)
    got = [_RequestState(r, p, 10, model, diffusion).base.seed for r, p in zip(reqs, plans)]
    assert got == want
    # eta = 0 draws nothing
    torch.manual_seed(99)
    _RequestState(replace(reqs[0], eta=0.0), plans[0], 10, model, diffusion)
    assert int(torch.randint(0, 2 ** 63 - 1, (1,), dtype=torch.int64).item()) == want[0]


# ------------------------------------------------------------------------------------------------
# DDIM requests in the batched paths (fake UNet, kernels restated in torch)
# ------------------------------------------------------------------------------------------------
def _ddim(k, S, eta, seed, **kw):
    return replace(_req(k, S, **kw), sampler="ddim", eta=eta, seed=seed)


def _alone_any(diffusion, req, scale=0.0):
    if req.sampler != "ddim":
        return _alone(diffusion, req, scale)
    req = _fresh(req)
    s = DDIMSampler(diffusion, FakeUNet(scale), alpha_generator_func=req.alpha_generator_func,
                    set_alpha_scale=set_alpha_scale)
    return s.sample(S=req.S, shape=(1, 4) + tuple(req.input["x"].shape[2:]), input=req.input, uc=req.uc,
                    guidance_scale=req.guidance_scale, eta=req.eta, seed=req.seed)


def test_ddim_alone_matches_the_restated_loop(diffusion, torch_kernels):
    """DDIMSampler on the fake UNet at eta = 0 equals cases_ddim.ddim_sample (ddim.py:63-131) on the same eps; at
    eta > 0 the seed fixes the latent."""
    req = _ddim(40, 10, 0.0, None)
    got = _alone_any(diffusion, req)
    swapped = []

    def eval_fn(inp, alpha):  # FakeUNet's eps at fuser scale alpha, with the SD1.5 conv from the first alpha 0 on
        swapped.append(alpha == 0)
        return (0.1 * inp["x"] + 1e-4 * inp["timesteps"].float().view(-1, 1, 1, 1) + 0.01 * inp["context"].mean()
                + 0.02 * float(alpha) + 0.03 * float(any(swapped)))

    want = CD.ddim_sample(eval_fn, _fresh(req).input, req.uc, 10, req.guidance_scale, alpha_type=[0.8, 0.0, 0.2])
    assert torch.allclose(got, want, rtol=1e-5, atol=1e-6)
    a, b = _alone_any(diffusion, _ddim(40, 10, 1.0, 5)), _alone_any(diffusion, _ddim(40, 10, 1.0, 5))
    assert torch.equal(a, b) and not torch.allclose(a, _alone_any(diffusion, _ddim(40, 10, 1.0, 6)))
    assert not torch.allclose(a, got)


@pytest.mark.parametrize("S", [10, 11])
def test_sample_requests_mixes_ddim_and_plms(diffusion, torch_kernels, S):
    reqs = [_req(31, S), _ddim(32, S, 0.0, None), _ddim(33, S, 0.7, 1234), _req(34, S, n=2, mis=0.36),
            _ddim(35, S, 0.7, 2 ** 40 + 1, alpha=None)]
    model = FakeUNet(scale=0.5)
    got = sample_requests(model, diffusion, [_fresh(r) for r in reqs], S, max_batch=8)
    # images evaluated: cond + uncond per trajectory and step, and the corrector's evaluation of the first step for
    # the PLMS requests only (the MIS request has 3 trajectories before its merge)
    steps = schedule_steps(S)
    merge = int(steps * 0.36)
    want = 2 * (steps + 1) + 3 * 2 * steps + 6 * (merge + 1) + 2 * (steps - merge)
    assert sum(sum(c["sizes"]) for c in model.calls) == want
    for k, r in enumerate(reqs):
        assert torch.allclose(got[k], _alone_any(diffusion, r, scale=0.5), rtol=1e-5, atol=1e-6), k


def test_engine_retires_ddim_after_steps_ticks(diffusion, torch_kernels):
    for eta, seed in ((0.0, None), (0.7, 77)):
        model = FakeUNet()
        eng = SamplingEngine(model, diffusion, buckets=None)
        req = _ddim(41, 11, eta, seed)
        finished, tick = {}, 0
        while tick <= 2 or eng.queued or eng.live:
            if tick == 2:
                eng.submit(_fresh(req))
            for t, x in eng.step().items():
                finished[t] = (tick, x)
            tick += 1
        steps = schedule_steps(11)
        assert finished[0][0] == 2 + steps - 1 and len(model.calls) == steps
        ts = [c["t"][0] for c in model.calls]
        assert ts == sorted(ts, reverse=True) and len(set(ts)) == steps
        assert torch.allclose(finished[0][1], _alone_any(diffusion, req), rtol=1e-5, atol=1e-6)


def test_engine_mixes_staggered_ddim_and_plms(diffusion, torch_kernels):
    model = FakeUNet()
    eng = SamplingEngine(model, diffusion, max_batch=8)
    arrivals = {0: [_ddim(50, 10, 0.7, 9), _req(51, 10, n=2, mis=0.36)], 3: [_ddim(52, 20, 0.0, None), _req(53, 11)],
                6: [_ddim(54, 11, 1.0, 10, alpha=None)]}
    out, reqs, tick = {}, {}, 0
    while tick <= max(arrivals) or eng.queued or eng.live:
        for r in arrivals.get(tick, []):
            reqs[eng.submit(_fresh(r))] = r
        out.update(eng.step())
        tick += 1
    assert set(out) == set(reqs)
    for t, r in reqs.items():
        assert torch.allclose(out[t], _alone_any(diffusion, r), rtol=1e-5, atol=1e-6), t
