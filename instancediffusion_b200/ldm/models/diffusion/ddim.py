"""DDIMSampler -- drop-in for ldm/models/diffusion/ddim.py (same constructor, `make_schedule` and `sample`).

GPU-first restructuring of `p_sample_ddim` (ddim.py:106-131), on the machinery of the PLMS samplers (`PLMSBase`):
  * the conditional and unconditional UNet evaluations are ONE batched forward (`PLMSBase._eval`) instead of two;
  * classifier-free guidance, the x_0 prediction, the x_{t-1} update and the eta noise are one fused kernel
    (idiff_ddim_update) instead of ~10 elementwise torch ops on the fp32 latent.

The eta noise comes from a counter-based generator inside the kernel: the noise of element i at schedule index `index`
is a function of (seed, index, i) only.  A run is reproduced from its integer seed, whatever else is batched with it
(`sample_requests`, `SamplingEngine`), and no generator state is carried between steps.

Documented differences from the reference:
  * at eta > 0 the reference draws `torch.randn_like` from the global CUDA generator, so its latents agree with these
    only in distribution; here `seed` (or, when None, one draw from torch's default CPU generator per `sample` call,
    which `torch.manual_seed` governs) fixes the noise;
  * the reference also calls `randn_like` at eta = 0 (multiplied by zero), which advances the CUDA generator; this
    sampler draws nothing at eta = 0.
"""
from __future__ import annotations

from typing import List, Optional

import numpy as np
import torch

from .... import ops
from ...modules.diffusionmodules.util import make_ddim_sampling_parameters
from ._plms_common import PLMSBase, Trajectory


def resolve_seed(eta: float, seed: Optional[int]) -> int:
    """The seed of a DDIM run: `seed` if given; at eta > 0 otherwise one draw from torch's default CPU generator;
    0 at eta = 0, where no noise is drawn (the generator is left untouched)."""
    if seed is not None:
        seed = int(seed)
        if not 0 <= seed < 1 << 64:
            raise ValueError(f"seed {seed} outside [0, 2^64)")
        return seed
    if eta == 0:
        return 0
    return int(torch.randint(0, 2 ** 63 - 1, (1,), dtype=torch.int64).item())


class DDIMBase(PLMSBase):
    """`PLMSBase` with the DDIM update: `make_schedule` keeps the eta sigmas, `_step_predict` has nothing to predict and
    `_step_finish` is one `ops.ddim_update` per trajectory, its noise keyed by (`self.seed`, index)."""

    seed = 0

    def make_schedule(self, ddim_num_steps, ddim_discretize="uniform", ddim_eta=0., verbose=False):
        """ddim.py:25-54: the schedule of `PLMSBase.make_schedule` and the sigmas of `ddim_eta` (util.py:73-83)."""
        if not ddim_eta >= 0:
            raise ValueError(f"ddim_eta must be >= 0, got {ddim_eta}")
        super().make_schedule(ddim_num_steps, ddim_discretize=ddim_discretize, ddim_eta=0., verbose=verbose)
        self.ddim_eta = float(ddim_eta)
        self.ddim_sigmas, _, _ = make_ddim_sampling_parameters(
            alphacums=self.diffusion.alphas_cumprod.detach().float().cpu(), ddim_timesteps=self.ddim_timesteps,
            eta=self.ddim_eta, verbose=verbose)

    def _step_predict(self, trajs: List[Trajectory], evals, ts_next, index, guidance_scale):
        """DDIM takes one evaluation per step."""
        return None

    def _step_finish(self, trajs: List[Trajectory], evals, pending, index, guidance_scale):
        """p_sample_ddim (ddim.py:110-131) after the evaluation at t, for every trajectory."""
        a_t, a_prev, _ = self._coefs(index)
        sigma = float(self.ddim_sigmas[index])
        gs = float(guidance_scale)
        for tr, (e_c, e_u) in zip(trajs, evals):
            x = tr.input["x"].float().contiguous()
            x_prev = torch.empty_like(x)
            ops.ddim_update(x, e_c, e_u, gs, a_t, a_prev, sigma, self.seed, index, None, x_prev)
            tr.input["x"] = x_prev


class DDIMSampler(DDIMBase):
    def __init__(self, diffusion, model, schedule="linear", alpha_generator_func=None, set_alpha_scale=None):
        super().__init__(diffusion, model, schedule, alpha_generator_func, set_alpha_scale)

    @torch.no_grad()
    def sample(self, S, shape, input, uc=None, guidance_scale=1, mask=None, x0=None, *, eta=0.0, seed=None):
        """ddim.py:57-60.  `input` is one input dict (there is no Multi-instance DDIM sampler).  eta > 0 adds the
        stochastic term of DDIM, its noise fixed by `seed` (see the module docstring)."""
        if not isinstance(input, dict):
            raise ValueError("DDIMSampler.sample takes one input dict; the Multi-instance input list is PLMS only "
                             "(PLMSSamplerInst)")
        self.make_schedule(ddim_num_steps=S, ddim_eta=eta)
        self.seed = resolve_seed(self.ddim_eta, seed)
        return self.ddim_sampling(shape, input, uc, guidance_scale, mask=mask, x0=x0)

    @torch.no_grad()
    def ddim_sampling(self, shape, input, uc, guidance_scale=1, mask=None, x0=None):
        """ddim.py:63-103."""
        b = shape[0]
        if input["x"] is None:
            input["x"] = torch.randn(shape, device=self.device)
        time_range = np.flip(self.ddim_timesteps)
        total_steps = self.ddim_timesteps.shape[0]
        alphas = self.alpha_generator_func(len(time_range)) if self.alpha_generator_func is not None else None
        tr = Trajectory(input)
        for i in range(len(time_range)):
            if alphas is not None:
                self._set_alpha(alphas[i])
            ts, ts_next = self._timesteps(b, i, time_range)
            if mask is not None:  # inpainting blend (ddim.py:94-98), as PLMSSampler
                assert x0 is not None
                img_orig = self.diffusion.q_sample(x0, ts)
                input["x"] = img_orig * mask + (1. - mask) * input["x"]
            self._step([tr], ts, ts_next, total_steps - i - 1, uc, guidance_scale)
        return input["x"]
