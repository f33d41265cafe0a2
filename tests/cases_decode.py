"""The image of a request, restated: the reference's post-processing of a decoded batch (inference.py:122-125, torch
on the device then numpy), the decode_to_image kernel restated in torch, and a fake first stage for the CPU tests of
the request drivers' `output="image"`."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from instancediffusion_b200.ldm.models.autoencoder import AutoencoderKL  # noqa: E402


def reference_post(x: torch.Tensor) -> np.ndarray:
    """inference.py:122-125 on every image of the decoder output x (B, 3, H, W): uint8 (B, H, W, 3)."""
    out = []
    for sample in x:
        sample = torch.clamp(sample, min=-1, max=1) * 0.5 + 0.5
        sample = sample.cpu().numpy().transpose(1, 2, 0) * 255
        out.append(sample.astype(np.uint8))
    return np.stack(out)


def restated_post(x: torch.Tensor) -> torch.Tensor:
    """idiff_decode_to_image in torch: uint8 (B, H, W, 3) = trunc((clamp(x, -1, 1) * 0.5 + 0.5) * 255) in fp32."""
    v = (torch.clamp(x.float(), -1, 1) * 0.5 + 0.5) * 255
    return v.trunc().to(torch.uint8).permute(0, 2, 3, 1).contiguous()


def decode_to_image(x, out):
    """ops.decode_to_image restated (its argument checks aside)."""
    return out.copy_(restated_post(x))


def fake_decode(z: torch.Tensor) -> torch.Tensor:
    """A stand-in decoder: (B, 4, h, w) -> (B, 3, 8h, 8w) fp32, per image, reaching past [-1, 1] so the clamp matters."""
    x = 1.5 * z[:, :3] + 0.1 * z[:, 3:]
    return x.repeat_interleave(8, dim=2).repeat_interleave(8, dim=3).contiguous()


class FakeAutoencoder:
    """`fake_decode` as the decoder under `AutoencoderKL.decode_images`; logs the batch of every decode."""

    decode_images = AutoencoderKL.decode_images

    def __init__(self):
        self.calls = []

    def decode(self, z):
        self.calls.append(z.shape[0])
        return fake_decode(z)
