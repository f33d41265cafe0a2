"""Inpainting requests restated for the tests: the blend in torch, the seeded q_sample the samplers are compared with,
the pixel-to-latent mask reduction, and the reference-golden cases.

* `inpaint_blend`: idiff_inpaint_blend in torch (same arguments as ops.inpaint_blend), what the CPU tests run instead of
  the kernel; `inpaint_blend64` the same in float64 for the kernel tests.
* `seeded_q_sample(diffusion, seed)`: `diffusion.q_sample` with its noise from the inpainting stream of cases_noise at
  the timestep, the function the samplers' mask / x0 blend is patched with to compare them with inpainting requests.
* `keep_of(repaint)`: a latent cell is kept when no pixel of its 8x8 block is to be repainted.
* `INPAINT_CASES`: the reference's PLMSSampler / DDIMSampler (eta 0) with mask / x0 on the seeded UNet of
  cases.UNET_CASE; tools/make_golden_inpaint.py writes tests/golden/inpaint.pt.
"""
from __future__ import annotations

import numpy as np
import torch

import cases_noise as CN

# name -> spec; the UNet, flavour and 64x64 latent are those of cases.UNET_CASE.  `box` is the repainted pixel box
# (y0, y1, x0, x1) of the 512x512 image, `src_seed` seeds the source latent x_init, `seed` the blend / start noise.
INPAINT_CASES = {
    "plms_S4": dict(sampler="plms", S=4, n=1, batch=1, seed=71, src_seed=81, input_seed=61, guidance=7.5,
                    alpha_type=[0.8, 0.0, 0.2], box=(96, 352, 128, 416)),
    "ddim_S10_b2": dict(sampler="ddim", S=10, n=2, batch=2, seed=72, src_seed=82, input_seed=62, guidance=7.5,
                        alpha_type=[0.8, 0.0, 0.2], box=(203, 461, 37, 300)),  # crosses alpha 0, unaligned box
}


def keep_of(repaint: torch.Tensor) -> torch.Tensor:
    """uint8 (Bm, H, W) keep mask of a (Bm, 8H, 8W) pixel repaint mask."""
    bm, h8, w8 = repaint.shape
    r = repaint.reshape(bm, h8 // 8, 8, w8 // 8, 8).ne(0).sum((2, 4))
    return (r == 0).to(torch.uint8)


def box_mask(b: int, size: int, box, dtype=torch.bool) -> torch.Tensor:
    """(b, size, size) repaint mask: True inside the pixel box (y0, y1, x0, x1)."""
    m = torch.zeros((b, size, size), dtype=torch.bool)
    y0, y1, x0, x1 = box
    m[:, y0:y1, x0:x1] = True
    return m.to(dtype)


def q_value(x0: torch.Tensor, sqrt_a: float, sqrt_1m_a: float, seed: int, t: int, shape) -> torch.Tensor:
    """sqrt_a * x0 + sqrt_1m_a * z over `shape` (x0 broadcast), in x0's dtype, z rounded to it first."""
    n = int(np.prod(shape))
    z = torch.from_numpy(CN.normals(seed, CN.INPAINT, t, n)).view(tuple(shape)).to(x0.device, x0.dtype)
    return sqrt_a * x0.expand(tuple(shape)) + sqrt_1m_a * z


def inpaint_blend(xs, outs, x0, keep, a, seed, t):
    """idiff_inpaint_blend in torch (same arguments as ops.inpaint_blend)."""
    shape = tuple(xs[0].shape)
    q = q_value(x0, float(a[0]), float(a[1]), seed, int(t), shape)
    k = keep.bool()[:, None]
    for x, o in zip(xs, outs):
        o.copy_(torch.where(k, q, x))
    return outs


def inpaint_blend64(xs, x0, keep, a, seed, t):
    """The blend of every x of xs in float64 on the CPU."""
    x0 = x0.detach().double().cpu()
    q = q_value(x0, float(a[0]), float(a[1]), seed, int(t), tuple(xs[0].shape))
    k = keep.cpu().bool()[:, None]
    return [torch.where(k, q, x.detach().double().cpu()) for x in xs]


def seeded_q_sample(diffusion, seed: int):
    """`diffusion.q_sample(x0, t)` with the blend's noise keyed by (seed, t) in place of torch.randn_like: the blend of
    an inpainting request, so a sampler's mask / x0 run with it is what the request drivers compute."""
    def q_sample(x_start, t, noise=None):
        assert noise is None
        tt = int(t.reshape(-1)[0])
        assert bool((t == tt).all())
        sa = float(diffusion.sqrt_alphas_cumprod[tt])
        s1m = float(diffusion.sqrt_one_minus_alphas_cumprod[tt])
        return q_value(x_start, sa, s1m, seed, tt, tuple(x_start.shape))
    return q_sample
