"""Image-to-image sampling (SDEdit) restated for the tests: the start step, the start-noise stream of idiff_noise_latent
in numpy, the start latent in float64 and in torch, and the PLMS / DDIM loops from the start step k0 in torch.

* `start_step(N, strength)`: k0 = N - int(N * strength); n_run = int(N * strength) must be >= 1.
* `x_start64` / `noise_latent`: sqrt(a) * x_init + sqrt(1 - a) * z in float64, z the start-noise stream of
  cases_noise, and in torch with ops.noise_latent's arguments (what the CPU tests run instead of the kernel).
* `plms_tail` / `ddim_tail`: the samplers' loops over steps k0 .. N-1 (plms.py:72-167, plms_instance.py:65-212,
  ddim.py:63-131), with the Multi-instance rule of a truncated schedule: trajectories merge before int(N * mis) only if
  that step lies after k0.
"""
from __future__ import annotations

from typing import Callable, List

import numpy as np
import torch

import cases_ddim as CD
import cases_noise as CN


def start_step(steps: int, strength: float) -> int:
    n_run = int(steps * strength)
    if not 0 < strength <= 1 or n_run < 1:
        raise ValueError(strength)
    return steps - n_run


def x_start64(x_init: torch.Tensor, a: float, seed: int, shape) -> torch.Tensor:
    """The start latent in float64 (CPU): x_init broadcast to `shape`."""
    n = int(np.prod(shape))
    z = torch.from_numpy(CN.normals(seed, CN.START, 0, n)).view(tuple(shape))
    x = x_init.detach().double().cpu().expand(tuple(shape))
    return a ** 0.5 * x + (1 - a) ** 0.5 * z


def noise_latent(x_init, a, seed, out):
    """idiff_noise_latent in torch (same arguments as ops.noise_latent)."""
    out.copy_(x_start64(x_init.reshape((-1,) + tuple(out.shape[1:])), float(a), seed, out.shape).to(out.dtype))
    return out


def _schedule(S: int):
    from oracle import torch_oracle as TO
    acp = TO.alphas_cumprod()
    steps = np.asarray(list(range(0, 1000, 1000 // S))) + 1
    a = acp[steps]
    a_prev = torch.tensor([acp[0].item()] + acp[steps[:-1]].tolist(), dtype=torch.float32)
    return acp, steps, a, a_prev


def start_latent(x_init: torch.Tensor, S: int, strength: float, seed: int, shape) -> tuple:
    """(k0, x_start in fp32 on x_init's device) for a schedule of S."""
    acp, steps, _, _ = _schedule(S)
    k0 = start_step(len(steps), strength)
    t0 = int(np.flip(steps)[k0])
    return k0, x_start64(x_init, float(acp[t0]), seed, shape).float().to(x_init.device)


def _alphas(total, alpha_type):
    from oracle import torch_oracle as TO
    return TO.alpha_schedule(total, alpha_type) if alpha_type is not None else [1] * total


def _model_out(eval_fn, inp, uc, guidance, alpha):
    e = eval_fn(inp, alpha)
    if uc is not None and guidance != 1:
        e_u = eval_fn(dict(x=inp["x"], timesteps=inp["timesteps"], context=uc), alpha)
        e = e_u + guidance * (e - e_u)
    return e


def plms_tail(eval_fn: Callable, inputs: List[dict], uc, S: int, guidance: float, x_start: torch.Tensor, k0: int,
              mis: float = 0.0, alpha_type=None) -> torch.Tensor:
    """eval_fn(input_dict, alpha) -> eps.  inputs: [global, inst_1 ..] (one entry without MIS), all started at
    x_start; steps k0 .. N-1 of PLMS, the first with the pseudo improved Euler predictor and corrector."""
    _, steps, a, a_prev = _schedule(S)
    time_range = np.flip(steps)
    total = len(steps)
    alphas = _alphas(total, alpha_type)
    merge = int(total * mis) if len(inputs) > 1 else None
    if merge is not None and merge <= k0:
        inputs, merge = inputs[:1], None
    for inp in inputs:
        inp["x"] = x_start

    def step(inp, old, i):
        index = total - i - 1
        b, dev = inp["x"].shape[0], inp["x"].device
        x = inp["x"].clone()
        t = torch.full((b,), int(time_range[i]), dtype=torch.long, device=dev)
        t_next = torch.full((b,), int(time_range[min(i + 1, total - 1)]), dtype=torch.long, device=dev)
        at, ap = float(a[index]), float(a_prev[index])

        def x_prev_of(e):
            return ap ** 0.5 * (x - (1. - at) ** 0.5 * e) / at ** 0.5 + (1. - ap) ** 0.5 * e

        inp["timesteps"] = t
        e_t = _model_out(eval_fn, inp, uc, guidance, alphas[i])
        if len(old) == 0:
            inp["x"] = x_prev_of(e_t)
            inp["timesteps"] = t_next
            e_p = (e_t + _model_out(eval_fn, inp, uc, guidance, alphas[i])) / 2
        elif len(old) == 1:
            e_p = (3 * e_t - old[-1]) / 2
        elif len(old) == 2:
            e_p = (23 * e_t - 16 * old[-1] + 5 * old[-2]) / 12
        else:
            e_p = (55 * e_t - 59 * old[-1] + 37 * old[-2] - 9 * old[-3]) / 24
        inp["x"] = x_prev_of(e_p)
        old.append(e_t)
        if len(old) >= 4:
            old.pop(0)

    olds = [[] for _ in inputs]
    for i in range(k0, total):
        if merge == i:
            inputs[0]["x"] = torch.stack([inp["x"] for inp in inputs]).mean(0)
            inputs, olds = inputs[:1], olds[:1]
        for inp, old in zip(inputs, olds):
            step(inp, old, i)
    if merge == total:
        inputs[0]["x"] = torch.stack([inp["x"] for inp in inputs]).mean(0)
    return inputs[0]["x"]


def ddim_tail(eval_fn: Callable, inp: dict, uc, S: int, guidance: float, x_start: torch.Tensor, k0: int,
              eta: float = 0.0, seed: int = 0, alpha_type=None) -> torch.Tensor:
    """Steps k0 .. N-1 of DDIM from x_start, the eta noise of step index `index` from cases_noise."""
    acp, steps, a, a_prev = _schedule(S)
    _, _, _, sig = CD.ddim_schedule(S, eta, acp)
    time_range = np.flip(steps)
    total = len(steps)
    alphas = _alphas(total, alpha_type)
    inp["x"] = x_start
    for i in range(k0, total):
        index = total - i - 1
        b = inp["x"].shape[0]
        inp["timesteps"] = torch.full((b,), int(time_range[i]), dtype=torch.long, device=inp["x"].device)
        e = _model_out(eval_fn, inp, uc, guidance, alphas[i])
        at, ap, s = float(a[index]), float(a_prev[index]), float(sig[index])
        x = ap ** 0.5 * (inp["x"] - (1. - at) ** 0.5 * e) / at ** 0.5 + max(1. - ap - s * s, 0.) ** 0.5 * e
        if s > 0:
            z = torch.from_numpy(CN.normals(seed, CN.DDIM_ETA, index, x.numel())).view_as(x).to(x.device, x.dtype)
            x = x + s * z
        inp["x"] = x
    return inp["x"]
