"""DPMSolverSampler -- DPM-Solver++(2M) with the other samplers' constructor and `sample` (not a reference module).

DPM-Solver++ in its second-order multistep form (Lu et al., "DPM-Solver++: Fast Solver for Guided Sampling of
Diffusion Probabilistic Models", 2022, Algorithm 2) on the data prediction x0 = (x - sigma_t e) / alpha_t, with
alpha = sqrt(a), sigma = sqrt(1 - a), lambda = log(alpha / sigma) and h_i = lambda_n - lambda_t per step:

    D      = x0_i                                              (the first step of a run)
    D      = (1 + 1/(2r)) x0_i - (1/(2r)) x0_{i-1},  r = h_{i-1} / h_i   (every later step)
    x_next = (sigma_n / sigma_t) x - alpha_n expm1(-h_i) D

One UNet evaluation per step.  With D = x0_i the update is DDIM's eta = 0 step, so the first step is exactly DDIM's.
The schedule is `PLMSBase.make_schedule(S)` ('uniform'), a_t / a_n the fp32 `ddim_alphas` / `ddim_alphas_prev` of the
step, so the last step goes to alphas_cumprod[0] as DDIM's does.  The scalars are computed in float64 on the host
(`dpmpp2m_coefs`) and the update runs as one fused kernel (idiff_dpmpp2m_update) per trajectory, CFG included.
No lower-order final step, SDE variant, thresholding or other timestep grid.
"""
from __future__ import annotations

import math
from typing import List, Optional, Tuple

import torch

from .... import ops
from ._plms_common import PLMSBase, Trajectory


def dpmpp2m_coefs(a_t: float, a_n: float, h_prev: Optional[float]) -> Tuple[float, ...]:
    """The scalars of one DPM-Solver++(2M) step from a_t to a_n (alphas_cumprod), in float64: (alpha_t, sigma_t,
    sigma_n / sigma_t, -alpha_n expm1(-h), w_cur, w_prev, h).  h_prev: the previous step's h, None on the first step
    of a run (then D = x0: w_cur = 1, w_prev = 0)."""
    alpha_t, sigma_t = math.sqrt(a_t), math.sqrt(1.0 - a_t)
    alpha_n, sigma_n = math.sqrt(a_n), math.sqrt(1.0 - a_n)
    h = math.log(alpha_n / sigma_n) - math.log(alpha_t / sigma_t)
    if h_prev is None:
        w_cur, w_prev = 1.0, 0.0
    else:
        r = h_prev / h
        w_cur, w_prev = 1.0 + 1.0 / (2.0 * r), -1.0 / (2.0 * r)
    return alpha_t, sigma_t, sigma_n / sigma_t, -alpha_n * math.expm1(-h), w_cur, w_prev, h


class DPMSolverBase(PLMSBase):
    """The DPM-Solver++(2M) sampler kind: `_step_finish`, the one update of a step, is one `ops.dpmpp2m_update` per
    trajectory, which keeps the step's x0 prediction and h as its `dpm_prev`."""
    sampler, title = "dpmpp_2m", "DPM-Solver++(2M)"
    eta_allowed, multi_instance, corrector_first = False, False, False

    def _step_finish(self, trajs: List[Trajectory], evals, pending, index, guidance_scale):
        a_t, a_n, _ = self._coefs(index)
        gs = float(guidance_scale)
        for tr, (e_c, e_u) in zip(trajs, evals):
            x = tr.input["x"].float().contiguous()
            x0_prev, h_prev = tr.dpm_prev if tr.dpm_prev is not None else (None, None)
            alpha_t, sigma_t, c_x, c_d, w_cur, w_prev, h = dpmpp2m_coefs(a_t, a_n, h_prev)
            x0 = torch.empty_like(x)
            x_next = torch.empty_like(x)
            ops.dpmpp2m_update(x, e_c, e_u, gs, x0_prev, alpha_t, sigma_t, c_x, c_d, w_cur, w_prev, x0, x_next)
            tr.input["x"] = x_next
            tr.dpm_prev = (x0, h)


class DPMSolverSampler(DPMSolverBase):
    """S steps of DPM-Solver++(2M) on one input dict (there is no Multi-instance DPM-Solver++ sampler), with the other
    samplers' constructor and `sample` (`PLMSBase.sample`): the alpha schedule, first-conv swap, mask / x0 blend and
    x_init / strength / seed.  The first step of an image-to-image run takes D = x0 as every first step does."""
