"""What the drop-in samplers send to the model, step by step, without a GPU: for every sampling step the
`set_alpha_scale` call and first-conv swap, and the multiset of UNet forwards (per input: batch, timestep, fuser scale,
first conv and which context it carries), against the log derived from the schedule.  Equal forwards keep the UNet's
CUDA-graph keys and hoisted-tensor cache hits, so this pins the samplers' speed as well as their model contract.  The
UNet is the fake of fake_unet.py and the kernels are restated in torch."""
import os
import sys
from dataclasses import replace

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from fake_unet import AGEN, FakeUNet, _fresh, _req, torch_kernels  # noqa: E402,F401
from test_img2img_cpu import _i2i  # noqa: E402
from instancediffusion_b200.ldm.models.diffusion.ddim import DDIMSampler  # noqa: E402
from instancediffusion_b200.ldm.models.diffusion.dpm_solver import DPMSolverSampler  # noqa: E402
from instancediffusion_b200.ldm.models.diffusion.plms import PLMSSampler  # noqa: E402
from instancediffusion_b200.ldm.models.diffusion.plms_instance import PLMSSamplerInst  # noqa: E402
from instancediffusion_b200.ldm.modules.diffusionmodules.util import make_ddim_timesteps  # noqa: E402
from instancediffusion_b200.utils.model import set_alpha_scale  # noqa: E402

pytestmark = pytest.mark.usefixtures("torch_kernels")


@pytest.fixture
def diffusion():
    from instancediffusion_b200.ldm.models.diffusion.ldm import LatentDiffusion
    return LatentDiffusion(linear_start=0.00085, linear_end=0.012, timesteps=1000)


class LoggingUNet(FakeUNet):
    """FakeUNet that appends its first-conv swaps and forwards to `log`; a forward is logged as the sorted tuple of its
    inputs' (batch, timestep, fuser scale, SD1.5 conv, context tag), the tag naming the context by its position in
    the sampler's input (or "uc")."""

    def __init__(self, log, tags):
        super().__init__()
        self.log, self.tags = log, tags

    def restore_first_conv_from_SD(self):
        self.log.append(("swap",))
        super().restore_first_conv_from_SD()

    def forward_batched(self, inputs, **kw):
        assert not kw, "the drop-in samplers pass no per-image scales or conv flags"
        out = super().forward_batched(inputs)
        c = self.calls[-1]
        self.log.append(("fwd", tuple(sorted(zip(c["sizes"], c["t"], c["scales"], c["restored"],
                                                 [self.tags[id(i["context"])] for i in inputs])))))
        return out


def _by_step(log):
    """The log split at each alpha: [(alpha, swaps, sorted forwards)] per step."""
    steps = []
    for ev in log:
        if ev[0] == "alpha":
            steps.append([ev[1], 0, []])
        elif ev[0] == "swap":
            steps[-1][1] += 1
        else:
            steps[-1][2].append(ev[1])
    return [(a, n, sorted(f)) for a, n, f in steps]


def _run(diffusion, cls, req, max_group=None, monkeypatch=None, **kw):
    """The sampler's step log for `req` (fake_unet._req with AGEN)."""
    log = []
    req = _fresh(req)
    ins = req.input if isinstance(req.input, list) else [req.input]
    tags = {id(i["context"]): str(k) for k, i in enumerate(ins)}
    tags[id(req.uc)] = "uc"
    model = LoggingUNet(log, tags)

    def alpha(m, a):
        log.append(("alpha", float(a)))
        set_alpha_scale(m, a)
    if max_group is not None:
        monkeypatch.setenv("IDIFF_MIS_GROUP", str(max_group))
    s = cls(diffusion, model, alpha_generator_func=req.alpha_generator_func, set_alpha_scale=alpha, **kw)
    extra = {} if req.x_init is None else dict(x_init=req.x_init, strength=req.strength, seed=req.seed)
    if cls is DDIMSampler:
        extra.update(eta=req.eta, seed=req.seed)
    x = s.sample(S=req.S, shape=(1, 4, 64, 64), input=req.input, uc=req.uc, guidance_scale=req.guidance_scale, **extra)
    assert x.shape == (1, 4, 64, 64) and torch.isfinite(x).all()
    return _by_step(log)


def _expected(req, two_evals_first, max_group=None):
    """The log the schedule implies: per step from k0, the step's alpha, a swap at alpha 0, and one forward per group of
    at most `max_group` live trajectories (cond and uncond of each) at t, plus the same forwards at t_next for the
    corrector of a first PLMS step.  Inputs run at the step's alpha and, from the first alpha 0 on, the SD1.5 conv."""
    N = len(make_ddim_timesteps("uniform", req.S, 1000))
    t = [int(v) for v in np.flip(make_ddim_timesteps("uniform", req.S, 1000))]
    alphas = AGEN(N)
    k0 = 0 if req.x_init is None else N - int(N * req.strength)
    n = len(req.input) if isinstance(req.input, list) else 1
    merge = int(N * req.mis) if n > 1 else None
    if merge is not None and req.x_init is not None and merge <= k0:
        merge = None
    out, swapped = [], False
    for i in range(k0, N):
        a = float(alphas[i])
        swapped |= a == 0
        live = list(range(n)) if merge is not None and i < merge else [0]
        g = max_group or len(live)
        groups = [live[j:j + g] for j in range(0, len(live), g)]
        times = [t[i]] + ([t[min(i + 1, N - 1)]] if two_evals_first and i == k0 else [])
        fwds = [tuple(sorted(e for k in grp for e in ((1, tv, a, swapped, str(k)), (1, tv, a, swapped, "uc"))))
                for tv in times for grp in groups]
        out.append((a, int(a == 0), sorted(fwds)))
    return out


CASES = {
    "plms": (PLMSSampler, lambda: _req(1, 10), {}),
    "mis036": (PLMSSamplerInst, lambda: _req(2, 10, n=4, mis=0.36), dict(mis=0.36, max_group=2)),
    "mis1": (PLMSSamplerInst, lambda: _req(3, 10, n=2, mis=1.0), dict(mis=1.0)),
    "ddim_eta": (DDIMSampler, lambda: replace(_req(4, 11), sampler="ddim", eta=0.7, seed=5), {}),
    "dpm": (DPMSolverSampler, lambda: replace(_req(5, 11), sampler="dpmpp_2m"), {}),
    "plms_i2i": (PLMSSampler, lambda: _i2i(_req(6, 10), 0.6, 11), {}),
    "mis_i2i": (PLMSSamplerInst, lambda: _i2i(_req(7, 10, n=4, mis=0.36), 0.9, 12), dict(mis=0.36, max_group=2)),
    "ddim_i2i": (DDIMSampler, lambda: replace(_i2i(_req(8, 11), 0.6, 13), sampler="ddim", eta=0.7), {}),
    "dpm_i2i": (DPMSolverSampler, lambda: replace(_i2i(_req(9, 11), 0.6, 14), sampler="dpmpp_2m"), {}),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_forwards_per_step(diffusion, monkeypatch, case):
    cls, make, kw = CASES[case]
    req = make()
    kw = dict(kw)
    max_group = kw.pop("max_group", None)
    got = _run(diffusion, cls, req, max_group=max_group, monkeypatch=monkeypatch, **kw)
    want = _expected(req, two_evals_first=cls in (PLMSSampler, PLMSSamplerInst), max_group=max_group)
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, (case, i)
