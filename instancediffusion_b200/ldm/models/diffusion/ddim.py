"""DDIMSampler -- drop-in for ldm/models/diffusion/ddim.py (same constructor, `make_schedule` and `sample`).

GPU-first restructuring of `p_sample_ddim` (ddim.py:106-131), on the sampling run of the PLMS samplers
(`PLMSBase.sample_loop`, `SamplingRun`):
  * the conditional and unconditional UNet evaluations are ONE batched forward instead of two;
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

from typing import List

import torch

from .... import ops
from ...modules.diffusionmodules.util import make_ddim_sampling_parameters
from ._plms_common import PLMSBase, Trajectory


class DDIMBase(PLMSBase):
    """The DDIM sampler kind: `make_schedule` keeps the eta sigmas and `_step_finish`, the one update of a step, is one
    `ops.ddim_update` per trajectory, its noise keyed by (`self.seed`, index)."""
    sampler, title = "ddim", "DDIM"
    eta_allowed, multi_instance, corrector_first = True, False, False

    def make_schedule(self, ddim_num_steps, ddim_discretize="uniform", ddim_eta=0., verbose=False):
        """ddim.py:25-54: the schedule of `PLMSBase.make_schedule` and the sigmas of `ddim_eta` (util.py:73-83)."""
        if not ddim_eta >= 0:
            raise ValueError(f"ddim_eta must be >= 0, got {ddim_eta}")
        super().make_schedule(ddim_num_steps, ddim_discretize=ddim_discretize, ddim_eta=0., verbose=verbose)
        self.ddim_eta = float(ddim_eta)
        self.ddim_sigmas, _, _ = make_ddim_sampling_parameters(
            alphacums=self.diffusion.alphas_cumprod.detach().float().cpu(), ddim_timesteps=self.ddim_timesteps,
            eta=self.ddim_eta, verbose=verbose)

    def noisy(self) -> bool:
        return self.ddim_eta > 0

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
    @torch.no_grad()
    def sample(self, S, shape, input, uc=None, guidance_scale=1, mask=None, x0=None, *, eta=0.0, seed=None,
               x_init=None, strength=1.0):
        """ddim.py:57-60.  `input` is one input dict (there is no Multi-instance DDIM sampler).  eta > 0 adds the
        stochastic term of DDIM, its noise fixed by `seed` (see the module docstring).  x_init / strength start
        image-to-image sampling as in PLMSSampler.sample; `seed` keys that start noise too."""
        return self._sample(S, shape, input, uc, guidance_scale, mask, x0, x_init, strength, seed, eta=eta)

    def ddim_sampling(self, shape, input, uc, guidance_scale=1, mask=None, x0=None, k0=0):
        """ddim.py:63-103 (its inpainting blend is ddim.py:94-98), from step k0 on: `PLMSBase.sample_loop`."""
        return self.sample_loop(shape, input, uc, guidance_scale, mask=mask, x0=x0, k0=k0)
