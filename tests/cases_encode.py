"""Image-to-image from images, restated for the tests: the posterior noise stream of idiff_encode_posterior in numpy, the
seeded posterior in torch, and a fake first stage whose `encode_images` is torch-only, for the CPU tests of the request
drivers' `init_image`.

* `posterior(moments, scale, seeds, index)`: distributions.py:24-36 and autoencoder.py:31 with the posterior stream of
  cases_noise, float64.
* `FakeAutoencoder`: `AutoencoderKL.encode_images` over a torch stand-in encoder, plus the fake decoder of
  cases_decode; logs the batch of every encode.
"""
from __future__ import annotations

from typing import Sequence

import torch

import cases_decode as CDec
import cases_noise as CN
from instancediffusion_b200.ldm.models.autoencoder import AutoencoderKL, check_images

SCALE = 0.18215


def quant_conv64(h: torch.Tensor, w: torch.Tensor, bias: torch.Tensor) -> torch.Tensor:
    """quant_conv (1x1) in float64: (B, 8, h, w) -> (B, 8, h, w) moments."""
    return torch.einsum("ok,bkhw->bohw", w.double().reshape(8, 8), h.double()) + bias.double().view(1, 8, 1, 1)


def posterior(moments: torch.Tensor, scale: float, seeds: Sequence[int], index: Sequence[int]) -> torch.Tensor:
    """(mean + exp(0.5 clamp(logvar, -30, 20)) * eps) * scale in float64 on the CPU, image b's eps the posterior stream
    at (seeds[b], index[b])."""
    m = moments.detach().double().cpu()
    mean, logvar = m[:, :4], m[:, 4:].clamp(-30.0, 20.0)
    eps = torch.stack([torch.from_numpy(CN.normals(s, CN.POSTERIOR, i, mean[0].numel())).view(mean.shape[1:])
                       for s, i in zip(seeds, index)])
    return (mean + torch.exp(0.5 * logvar) * eps) * scale


def fake_moments(images: torch.Tensor) -> torch.Tensor:
    """A stand-in encoder: uint8 (B, H, W, 3) -> (B, 8, H/8, W/8) moments, per image, from the normalised image."""
    x = (images.float() / 127.5 - 1).permute(0, 3, 1, 2)
    p = torch.nn.functional.avg_pool2d(x, 8)
    mean = torch.cat([p, p.mean(1, keepdim=True)], 1)
    return torch.cat([mean, 0.5 * mean - 3.0], 1)


class FakeAutoencoder(CDec.FakeAutoencoder):
    """`AutoencoderKL.encode_images` on `fake_moments` and the restated posterior, next to the fake decoder; logs the
    batch of every encode in `encode_calls` and its (image size, seeds, index) in `encode_args`."""

    encode_images = AutoencoderKL.encode_images
    scale_factor = SCALE

    def __init__(self):
        super().__init__()
        self.encode_calls, self.encode_args = [], []

    def _encode_images(self, images, seeds, index):
        check_images(images)
        assert images.shape[0] == len(seeds) == len(index)
        self.encode_calls.append(images.shape[0])
        self.encode_args.append((tuple(images.shape[1:3]), [int(x) for x in seeds], [int(i) for i in index]))
        return posterior(fake_moments(images), SCALE, seeds, index).float()


def random_images(b: int, h: int, w: int, seed: int) -> torch.Tensor:
    """uint8 (b, h, w, 3), every byte value likely."""
    return torch.randint(0, 256, (b, h, w, 3), generator=torch.Generator().manual_seed(seed), dtype=torch.uint8)
