"""DPM-Solver++(2M) restated for the tests: the fused update in float64 torch (what the CPU tests run instead of
idiff_dpmpp2m_update), the sampler's loop from the start step k0, and the Gaussian-data model whose probability-flow ODE
has a closed-form solution.

* `dpmpp2m_update`: ops.dpmpp2m_update's arguments, the arithmetic in float64, the results stored in the outputs' dtype.
* `dpm_tail`: steps k0 .. N-1 of the schedule of S ('uniform', a_t = alphas_cumprod[t], a_n = that of the next
  timestep, alphas_cumprod[0] after the last), every scalar derived here in float64 from a_t and a_n:
  alpha = sqrt(a), sigma = sqrt(1 - a), lambda = log(alpha / sigma), h = lambda_n - lambda_t,
  x0 = (x - sigma_t e) / alpha_t, D = x0 on the first step of the run, else (1 + 1/(2r)) x0 - x0_prev / (2r) with
  r = h_prev / h, and x_next = (sigma_n / sigma_t) x - alpha_n expm1(-h) D.
* `gaussian_eps` / `gaussian_flow_end`: for data N(mu, s^2) the exact eps is sigma_t (x - alpha_t mu) / (alpha_t^2 s^2 +
  sigma_t^2), and the probability-flow ODE carries x_T at a_T to alpha_0 mu + sqrt(alpha_0^2 s^2 + sigma_0^2) (x_T -
  alpha_T mu) / sqrt(alpha_T^2 s^2 + sigma_T^2) at a_0: the standardised value is constant along the flow.
"""
from __future__ import annotations

import math
from typing import Callable

import numpy as np
import torch

import cases_img2img as CI


def dpmpp2m_update(x, e_c, e_u, gs, x0_prev, alpha_t, sigma_t, c_x, c_d, w_cur, w_prev, x0_out, x_out):
    """idiff_dpmpp2m_update in float64 torch (same arguments as ops.dpmpp2m_update)."""
    xd, e = x.double(), e_c.double()
    if e_u is not None:
        e = e_u.double() + gs * (e - e_u.double())
    x0 = (xd - sigma_t * e) / alpha_t
    d = w_cur * x0
    if x0_prev is not None:
        d = d + w_prev * x0_prev.double()
    if x0_out is not None:
        x0_out.copy_(x0)
    x_out.copy_(c_x * xd + c_d * d)


def dpm_tail(eval_fn: Callable, inp: dict, uc, S: int, guidance: float, x_start: torch.Tensor, k0: int = 0,
             alpha_type=None) -> torch.Tensor:
    """eval_fn(input_dict, alpha) -> eps.  Steps k0 .. N-1 of DPM-Solver++(2M) from x_start, in float64."""
    _, steps, a, a_prev = CI._schedule(S)
    time_range = np.flip(steps)
    total = len(steps)
    alphas = CI._alphas(total, alpha_type)
    inp["x"] = x_start
    x0_prev = h_prev = None
    for i in range(k0, total):
        index = total - i - 1
        b = inp["x"].shape[0]
        inp["timesteps"] = torch.full((b,), int(time_range[i]), dtype=torch.long, device=inp["x"].device)
        x = inp["x"].double()
        # the model sees the latent in fp32, as the sampler keeps it
        e = CI._model_out(eval_fn, dict(inp, x=x.float()), uc, guidance, alphas[i]).double()
        at, an = float(a[index]), float(a_prev[index])
        al_t, sg_t, al_n, sg_n = math.sqrt(at), math.sqrt(1 - at), math.sqrt(an), math.sqrt(1 - an)
        h = math.log(al_n / sg_n) - math.log(al_t / sg_t)
        x0 = (x - sg_t * e) / al_t
        if x0_prev is None:
            d = x0
        else:
            r = h_prev / h
            d = (1 + 1 / (2 * r)) * x0 - x0_prev / (2 * r)
        inp["x"] = (sg_n / sg_t) * x - al_n * math.expm1(-h) * d
        x0_prev, h_prev = x0, h
    return inp["x"]


def gaussian_eps(x: torch.Tensor, a: float, mu: float, s: float) -> torch.Tensor:
    """The exact eps of data N(mu, s^2) at alphas_cumprod a."""
    al, sg = math.sqrt(a), math.sqrt(1 - a)
    return sg * (x - al * mu) / (al * al * s * s + sg * sg)


def gaussian_flow_end(x_T: torch.Tensor, a_T: float, a_0: float, mu: float, s: float) -> torch.Tensor:
    """The probability-flow ODE's solution at a_0 from x_T at a_T, for data N(mu, s^2)."""
    def std(a):
        return math.sqrt(a * s * s + 1 - a)
    return math.sqrt(a_0) * mu + std(a_0) * (x_T.double() - math.sqrt(a_T) * mu) / std(a_T)
