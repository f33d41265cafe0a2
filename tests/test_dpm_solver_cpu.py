"""DPM-Solver++(2M) without a GPU: DPMSolverSampler against the float64 restatement of its loop (tests/cases_dpm.py),
its first step against DDIM's, request validation, DPM-Solver++ requests next to PLMS / DDIM / image-to-image ones in
`sample_requests` and `SamplingEngine`, and the solver's order of convergence on Gaussian data, whose probability-flow
ODE has a closed-form solution.  The UNet is the fake of fake_unet.py and the kernels are restated in torch."""
import math
import os
import sys
from dataclasses import replace

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import cases_dpm as CP  # noqa: E402
import cases_img2img as CI  # noqa: E402
from fake_unet import AGEN, FakeUNet, _fresh, _req, torch_kernels  # noqa: E402,F401
from test_img2img_cpu import ALPHA_TYPE, TOL, _eval_fn, _i2i  # noqa: E402
from test_img2img_cpu import _alone as _alone_other  # noqa: E402
from instancediffusion_b200.ldm.models.diffusion._plms_common import SamplingRun  # noqa: E402
from instancediffusion_b200.ldm.models.diffusion.batched import (  # noqa: E402
    RequestPlan, _RequestState, check_requests, sample_requests, schedule_steps)
from instancediffusion_b200.ldm.models.diffusion.ddim import DDIMBase, DDIMSampler  # noqa: E402
from instancediffusion_b200.ldm.models.diffusion.dpm_solver import DPMSolverBase, DPMSolverSampler  # noqa: E402
from instancediffusion_b200.ldm.models.diffusion.engine import SamplingEngine  # noqa: E402
from instancediffusion_b200.utils.model import set_alpha_scale  # noqa: E402


@pytest.fixture
def diffusion():
    from instancediffusion_b200.ldm.models.diffusion.ldm import LatentDiffusion
    return LatentDiffusion(linear_start=0.00085, linear_end=0.012, timesteps=1000)


def _dpm(req):
    return replace(req, sampler="dpmpp_2m")


def _alone(diffusion, req, scale=0.0):
    """The request through its own sampler on a fresh fake."""
    if req.sampler != "dpmpp_2m":
        return _alone_other(diffusion, req, scale)
    req = _fresh(req)
    s = DPMSolverSampler(diffusion, FakeUNet(scale), alpha_generator_func=req.alpha_generator_func,
                         set_alpha_scale=set_alpha_scale)
    new = {} if req.x_init is None else dict(x_init=req.x_init, strength=req.strength, seed=req.seed)
    return s.sample(S=req.S, shape=(1, 4) + tuple(req.input["x"].shape[2:]), input=req.input, uc=req.uc,
                    guidance_scale=req.guidance_scale, **new)


# ------------------------------------------------------------------------------------------------
# the sampler against the restated loop
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cfg", [True, False])
@pytest.mark.parametrize("alpha", [True, False])
@pytest.mark.parametrize("strength", [1.0, 0.6])
@pytest.mark.parametrize("S", [10, 11])
def test_sampler_matches_restated_loop(diffusion, torch_kernels, cfg, alpha, strength, S):
    req = _dpm(_req(80, S, alpha=AGEN if alpha else None))
    if not cfg:
        req = replace(req, uc=None, guidance_scale=1.0)
    if strength != 1.0:
        req = _i2i(req, strength, 2 ** 40 + 7)
    got = _alone(diffusion, req)
    N = schedule_steps(S)
    if req.x_init is None:
        k0, xs = 0, req.input["x"].clone()
    else:
        k0, xs = CI.start_latent(req.x_init, S, strength, req.seed, (1, 4, 64, 64))
    assert torch_kernels["dpmpp2m_update"] == N - k0  # one update, and one evaluation, per step
    # without an alpha schedule the fake runs at its fuser scale 0 and its own conv throughout
    def plain_eval(inp, _):
        return 0.1 * inp["x"] + 1e-4 * inp["timesteps"].float().view(-1, 1, 1, 1) + 0.01 * inp["context"].mean()
    eval_fn = _eval_fn() if alpha else plain_eval
    want = CP.dpm_tail(eval_fn, _fresh(req).input, req.uc, S, req.guidance_scale, xs, k0,
                       alpha_type=ALPHA_TYPE if alpha else None)
    assert got.dtype == torch.float32
    assert torch.allclose(got.double(), want, **TOL), (got.double() - want).abs().max().item()


def test_mask_blend(diffusion, torch_kernels, monkeypatch):
    """mask / x0 take the other samplers' host-level blend: before every evaluation the kept region is x0 noised to the
    step's timestep (q_sample, made deterministic here), and a zero mask leaves the run as it is without one."""
    req = _dpm(_req(81, 10))
    x0 = torch.randn((1, 4, 64, 64), generator=torch.Generator().manual_seed(3))
    monkeypatch.setattr(diffusion, "q_sample", lambda x_start, t: x_start * (t.float().view(-1, 1, 1, 1) + 1))
    seen = []

    class Recording(FakeUNet):
        def forward_batched(self, inputs, **kw):
            seen.append((int(inputs[0]["timesteps"][0]), [i["x"].clone() for i in inputs]))
            return super().forward_batched(inputs, **kw)

    def run(mask):
        r = _fresh(req)
        s = DPMSolverSampler(diffusion, Recording(), alpha_generator_func=r.alpha_generator_func,
                             set_alpha_scale=set_alpha_scale)
        return s.sample(10, (1, 4, 64, 64), r.input, uc=r.uc, guidance_scale=r.guidance_scale, mask=mask, x0=x0)
    mask = torch.zeros((1, 4, 64, 64))
    mask[..., :32] = 1
    run(mask)
    assert len(seen) == schedule_steps(10)
    for t, xs in seen:
        for x in xs:  # cond and uncond
            assert torch.equal(x[..., :32], (x0 * float(t + 1))[..., :32]), t
    assert torch.equal(run(torch.zeros((1, 4, 64, 64))), _alone(diffusion, req))


# ------------------------------------------------------------------------------------------------
# the first step is DDIM's
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k0", [0, 4])
def test_first_run_step_equals_ddim(diffusion, torch_kernels, k0):
    """x_next with D = x0 is sqrt(a_n) x0 + sqrt(1 - a_n) e: the first step of a run (also one from k0 > 0) equals
    DDIM's at eta = 0.  The second step differs: it adds the correction from the first step's x0."""
    S, gs = 10, 7.5
    req = _req(82, S)
    outs = {}
    for cls in (DPMSolverBase, DDIMBase):
        base = cls(diffusion, FakeUNet())
        base.make_schedule(S)
        run = SamplingRun(base, [dict(_fresh(req).input)], (1, 4, 64, 64), RequestPlan(1, None, 1, True, k0), gs, None)
        run.start()
        xs = []
        for i in (k0, k0 + 1):  # one step of the drop-in samplers' loop
            run.begin()
            run.advance(base._forward(run, req.uc))
            assert run.i == i + 1
            xs.append(run.trajs[0].input["x"].clone())
        outs[cls] = xs
    (d1, d2), (g1, g2) = outs[DPMSolverBase], outs[DDIMBase]
    assert torch.allclose(d1, g1, **TOL), (d1 - g1).abs().max().item()
    assert not torch.allclose(d2, g2, rtol=1e-3, atol=1e-4)


# ------------------------------------------------------------------------------------------------
# validation
# ------------------------------------------------------------------------------------------------
def test_validation(diffusion):
    ok = _dpm(_req(83, 10))
    assert check_requests([ok], 10, 32) == [RequestPlan(1, None, 1, True)]
    assert check_requests([_i2i(ok, 0.35, 1)], 10, 32) == [RequestPlan(1, None, 1, True, 7)]
    with pytest.raises(ValueError, match=r"request 0: eta=0.5 needs sampler='ddim' \(DPM-Solver\+\+\(2M\) is"):
        check_requests([replace(ok, eta=0.5)], 10, 32)
    multi = _dpm(_req(84, 10, n=2, mis=0.36))
    with pytest.raises(ValueError, match=r"DPM-Solver\+\+\(2M\) takes one input dict .* PLMS only"):
        check_requests([multi], 10, 32)
    with pytest.raises(ValueError, match="PLMS only"):
        check_requests([replace(multi, mis=0.0)], 10, 32)
    with pytest.raises(ValueError, match="PLMS only"):
        check_requests([replace(ok, mis=0.36)], 10, 32)
    for bad in ("dpm", "dpmpp_2s", "DPMPP_2M"):
        with pytest.raises(ValueError, match="unknown sampler"):
            check_requests([replace(ok, sampler=bad)], 10, 32)
    eng = SamplingEngine(FakeUNet(), diffusion)
    assert eng.submit(_fresh(ok)) == 0
    for bad in (replace(ok, eta=0.5), multi, replace(ok, sampler="dpm")):
        with pytest.raises(ValueError):
            eng.submit(bad)
    with pytest.raises(ValueError, match="input dict"):
        DPMSolverSampler(diffusion, FakeUNet()).sample(10, (1, 4, 64, 64), multi.input)
    # no noise without x_init: an unseeded request draws nothing; one from x_init draws its start-noise seed
    torch.manual_seed(99)
    want = int(torch.randint(0, 2 ** 63 - 1, (1,), dtype=torch.int64).item())
    torch.manual_seed(99)
    assert _RequestState(ok, check_requests([ok], 10, 32)[0], 10, FakeUNet(), diffusion).base.seed == 0
    i2i, model = _i2i(ok, 0.5, None), FakeUNet()
    torch.manual_seed(99)
    assert _RequestState(i2i, check_requests([i2i], 10, 32)[0], 10, model, diffusion).base.seed == want


# ------------------------------------------------------------------------------------------------
# the request drivers
# ------------------------------------------------------------------------------------------------
def _mix(S):
    """DPM-Solver++ requests (plain, without alpha schedule, without CFG, image-to-image at two strengths) next to
    PLMS, DDIM, Multi-instance and image-to-image PLMS requests."""
    return [
        _dpm(_req(90, S)),
        _req(91, S),
        replace(_req(92, S), sampler="ddim", eta=0.7, seed=5),
        _dpm(_req(93, S, alpha=None)),
        _req(94, S, n=2, mis=0.36),
        _dpm(_i2i(_req(95, S), 0.6, 31)),
        _i2i(_req(96, S), 0.35, 32),
        replace(_dpm(_req(97, S)), uc=None, guidance_scale=1.0),
        _dpm(_i2i(_req(98, S), 0.35, 33)),
    ]


def _images(req, S):
    """Images a request evaluates in a whole run: cond (+ uncond) per live trajectory and step from k0, and the
    corrector's evaluation of a first PLMS step."""
    N = schedule_steps(S)
    k0 = 0 if req.x_init is None else N - int(N * req.strength)
    n = len(req.input) if isinstance(req.input, list) else 1
    merge = int(N * req.mis) if n > 1 else None

    def live(i):
        return n if merge is not None and i < merge else 1
    rows = 2 if req.uc is not None and req.guidance_scale != 1 else 1
    return rows * (sum(live(i) for i in range(k0, N)) + (live(k0) if req.sampler == "plms" else 0))


@pytest.mark.parametrize("S", [10, 11])
def test_sample_requests_mixes_dpm_requests(diffusion, torch_kernels, S):
    reqs = _mix(S)
    model = FakeUNet(scale=0.5)
    got = sample_requests(model, diffusion, [_fresh(r) for r in reqs], S, max_batch=8)
    assert sum(sum(c["sizes"]) for c in model.calls) == sum(_images(r, S) for r in reqs)
    for k, r in enumerate(reqs):
        assert torch.allclose(got[k], _alone(diffusion, r, scale=0.5), **TOL), k


def test_engine_retires_dpm_after_n_run_ticks(diffusion, torch_kernels):
    for strength in (1.0, 0.6, 0.35):
        model = FakeUNet()
        eng = SamplingEngine(model, diffusion, buckets=None)
        req = _dpm(_req(99, 11)) if strength == 1.0 else _dpm(_i2i(_req(99, 11), strength, 41))
        finished, tick = {}, 0
        while tick <= 2 or eng.queued or eng.live:
            if tick == 2:
                eng.submit(_fresh(req))
            for t, x in eng.step().items():
                finished[t] = (tick, x)
            tick += 1
        n_run = int(schedule_steps(11) * strength)
        assert finished[0][0] == 2 + n_run - 1 and len(model.calls) == n_run, strength
        ts = [c["t"][0] for c in model.calls]
        assert ts == sorted(ts, reverse=True) and len(set(ts)) == n_run
        assert torch.allclose(finished[0][1], _alone(diffusion, req), **TOL)


def test_engine_mixes_staggered_dpm_requests(diffusion, torch_kernels):
    model = FakeUNet()
    eng = SamplingEngine(model, diffusion, max_batch=8)
    mix = [replace(r, S=S) for r, S in zip(_mix(10), (10, 11, 10, 20, 10, 11, 10, 25, 20))]
    arrivals = {0: mix[:3], 2: mix[3:5], 4: mix[5:7], 7: mix[7:]}
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
        n_run = int(schedule_steps(r.S) * r.strength)
        assert done_at[t] - sub_at[t] + 1 == n_run + (r.sampler == "plms"), t  # admitted at once: live images fit
    evaluated = sum(sum(c["sizes"]) for c in model.calls) - eng.padded_images
    assert evaluated == sum(_images(r, r.S) for r in reqs.values())


# ------------------------------------------------------------------------------------------------
# order of convergence on Gaussian data
# ------------------------------------------------------------------------------------------------
MU, STD = 0.7, 0.5


class GaussianEps:
    """The exact eps of data N(MU, STD^2) at the timesteps of the input, from the fp32 alphas_cumprod the samplers
    read (no forward_batched: the samplers evaluate it as a plain model)."""

    def __init__(self, diffusion):
        self.acp = diffusion.alphas_cumprod.float()

    def __call__(self, inp):
        a = float(self.acp[int(inp["timesteps"][0])])
        return CP.gaussian_eps(inp["x"].double(), a, MU, STD).float()


def _flow_error(diffusion, cls, S):
    """RMS error of the sampler's end point against the ODE's closed-form end point, over 20 000 samples."""
    x_T = torch.randn((1, 4, 50, 100), generator=torch.Generator().manual_seed(0))
    s = cls(diffusion, GaussianEps(diffusion))
    got = s.sample(S, tuple(x_T.shape), dict(x=x_T.clone(), timesteps=None, context=None))
    acp = diffusion.alphas_cumprod.float()
    a_T = float(acp[int(s.ddim_timesteps[-1])])
    want = CP.gaussian_flow_end(x_T, a_T, float(acp[0]), MU, STD)
    return (got.double() - want).pow(2).mean().sqrt().item()


def test_convergence_order(diffusion, torch_kernels):
    """DPM-Solver++(2M) converges at second order on the 'uniform' grids (observed order >= 1.4 over S = 100 -> 200 ->
    500; a wrong r, sign or stale history drops it to 1), DDIM at first order (<= 1.1), and DPM-Solver++ is the more
    accurate of the two at every S tested."""
    err = {cls: {S: _flow_error(diffusion, cls, S) for S in (10, 20, 50, 100, 200, 500)}
           for cls in (DPMSolverSampler, DDIMSampler)}
    order = {cls: [math.log(e[a] / e[b]) / math.log(b / a) for a, b in ((100, 200), (200, 500))]
             for cls, e in err.items()}
    print(f"[convergence] DPM-Solver++(2M) errors {err[DPMSolverSampler]} orders {order[DPMSolverSampler]}")
    print(f"[convergence] DDIM errors {err[DDIMSampler]} orders {order[DDIMSampler]}")
    assert min(order[DPMSolverSampler]) >= 1.4, order
    assert max(order[DDIMSampler]) <= 1.1, order
    for S in (10, 20, 50, 100):
        assert err[DPMSolverSampler][S] < err[DDIMSampler][S], S
