"""Seeded DDIM cases (tests/golden/ddim.pt) and the plain-torch / numpy restatements the DDIM tests check against.

* `DDIM_CASES`: the reference's DDIMSampler.sample at eta = 0 on the seeded UNet of cases.UNET_CASE (64x64 latent, CFG
  7.5, alpha type [0.8, 0.0, 0.2]); tools/make_golden_ddim.py writes the latents, the GPU tests compare the mirror with
  them and the CPU tests compare `ddim_sample` with them.
* `ddim_update`: idiff_ddim_update restated in torch with its noise from cases_noise (what the CPU scheduling tests run
  instead of the kernel).
* `ddim_sample`: ddim.py:63-131 at eta = 0 restated in torch (the DDIM counterpart of torch_oracle.plms_sample).
"""
from __future__ import annotations

from typing import Callable

import numpy as np
import torch

import cases_noise as CN

# name -> spec; the UNet, flavour and latent size are those of cases.UNET_CASE
DDIM_CASES = {
    "ddim_S4": dict(S=4, n=1, batch=1, seed=61, guidance=7.5, alpha_type=[0.8, 0.0, 0.2]),
    "ddim_S10_b2": dict(S=10, n=2, batch=2, seed=62, guidance=7.5, alpha_type=[0.8, 0.0, 0.2]),  # crosses alpha 0
}

def ddim_update(x, e_c, e_u, gs, a_t, a_prev, sigma, seed, index, e_out, x_out):
    """idiff_ddim_update in torch (same arguments as ops.ddim_update)."""
    e = e_c if e_u is None else e_u + gs * (e_c - e_u)
    pred_x0 = (x - (1 - a_t) ** 0.5 * e) / a_t ** 0.5
    xp = a_prev ** 0.5 * pred_x0 + max(1 - a_prev - sigma ** 2, 0.0) ** 0.5 * e
    if sigma > 0:
        z = torch.from_numpy(CN.normals(seed, CN.DDIM_ETA, index, x.numel())).to(x.dtype).view_as(x)
        xp = xp + sigma * z
    if e_out is not None:
        e_out.copy_(e)
    x_out.copy_(xp)


# ------------------------------------------------------------------------------------------------
# ddim.py:25-54 (schedule) and 63-131 (sampling loop) at eta = 0
# ------------------------------------------------------------------------------------------------
def ddim_schedule(S: int, eta: float, acp: torch.Tensor):
    """util.py:48-83 in float64 from the fp32 alphas_cumprod: (timesteps, alphas, alphas_prev, sigmas).  1 - alphas is
    rounded to fp32 first, as the reference computes it on its fp32 tensor before numpy promotes the quotient."""
    steps = np.asarray(list(range(0, 1000, 1000 // S))) + 1
    a = acp.double().numpy()
    alphas = a[steps]
    alphas_prev = np.asarray([a[0]] + a[steps[:-1]].tolist())
    one_minus = (1 - acp[steps].float()).double().numpy()
    sigmas = eta * np.sqrt((1 - alphas_prev) / one_minus * (1 - alphas / alphas_prev))
    return steps, alphas, alphas_prev, sigmas


def ddim_sample(eval_fn: Callable, input: dict, uc, S: int, guidance: float, alpha_type=None):
    """eval_fn(input_dict, alpha) -> eps.  DDIMSampler.sample at eta = 0 (ddim.py:63-131): no noise term."""
    from oracle import torch_oracle as TO
    acp = TO.alphas_cumprod()
    steps = np.asarray(list(range(0, 1000, 1000 // S))) + 1
    a = acp[steps]
    a_prev = torch.tensor([acp[0].item()] + acp[steps[:-1]].tolist(), dtype=torch.float32)
    time_range = np.flip(steps)
    total = len(steps)
    alphas = TO.alpha_schedule(total, alpha_type) if alpha_type is not None else [1] * total
    inp = input
    for i, step in enumerate(time_range):
        index = total - i - 1
        b = inp["x"].shape[0]
        inp["timesteps"] = torch.full((b,), int(step), dtype=torch.long, device=inp["x"].device)
        e = eval_fn(inp, alphas[i])
        if uc is not None and guidance != 1:
            e_u = eval_fn(dict(x=inp["x"], timesteps=inp["timesteps"], context=uc), alphas[i])
            e = e_u + guidance * (e - e_u)
        at, ap = a[index], a_prev[index]
        pred_x0 = (inp["x"] - torch.sqrt(1. - at) * e) / at.sqrt()
        inp["x"] = ap.sqrt() * pred_x0 + (1. - ap).sqrt() * e
    return inp["x"]


def ref_inputs_for(gti, name: str, device="cpu") -> tuple:
    """(input dict, uc) of a case, built like cases.SAMPLER_CASES inputs."""
    from instancediffusion_b200 import synthetic
    sc = DDIM_CASES[name]
    return synthetic.make_sampler_inputs(gti, sc["batch"], sc["n"], sc["seed"], "box", mis=False, device=device)
