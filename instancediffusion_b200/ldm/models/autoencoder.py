"""First-stage model of the sampling pipeline: `AutoencoderKL.decode` turns the denoised latent into the
image right after the sampler loop (inference.py:96).  Same class name, constructor signature and
state_dict keys as the reference's ldm/models/autoencoder.py:12-37 (loaded strict by
utils/checkpoint.py:233), with the arithmetic in libidiff_b200.so.

decode(z) = Decoder(post_quant_conv(z / scale_factor)): the scale, the 1x1 post_quant_conv and the
NCHW fp32 -> NHWC fp16 conversion are one kernel (idiff_vae_latent_in); everything after it is the GEMM /
GroupNorm kernels of the UNet (ldm/modules/diffusionmodules/model.py in this package).

encode_images(images, seed) = posterior.sample() * scale_factor of uint8 images: conv_in reads the bytes
(idiff_encode_image_in), quant_conv and the sample are one kernel (idiff_encode_posterior) whose noise is keyed by
(seed, image index) instead of drawn from torch's global generator.
"""
from __future__ import annotations

import torch

from ... import ops
from .diffusion._plms_common import resolve_seed
from ..modules._base import PackedModule, f32
from ..modules.diffusionmodules.model import Decoder, Encoder


class DiagonalGaussianDistribution(object):
    """ldm/modules/distributions/distributions.py:24-41 (the part `encode` uses)."""

    def __init__(self, parameters, deterministic=False):
        self.parameters = parameters
        self.mean, self.logvar = torch.chunk(parameters, 2, dim=1)
        self.logvar = torch.clamp(self.logvar, -30.0, 20.0)
        self.deterministic = deterministic
        self.std = torch.exp(0.5 * self.logvar)
        self.var = torch.exp(self.logvar)
        if self.deterministic:
            self.var = self.std = torch.zeros_like(self.mean)

    def sample(self):
        return self.mean + self.std * torch.randn(self.mean.shape).to(device=self.parameters.device)

    def mode(self):
        return self.mean


def check_images(images, multiple: int = 8) -> None:
    """uint8 (B, H, W, 3) with B >= 1 and H, W positive multiples of `multiple`, or ValueError."""
    if not isinstance(images, torch.Tensor) or images.dtype != torch.uint8:
        raise ValueError(f"images must be a uint8 tensor, got {getattr(images, 'dtype', type(images))}")
    if images.dim() != 4 or images.shape[-1] != 3 or images.shape[0] < 1:
        raise ValueError(f"images must be (B, H, W, 3) RGB, got shape {tuple(images.shape)}")
    H, W = int(images.shape[1]), int(images.shape[2])
    if H < 1 or W < 1 or H % multiple or W % multiple:
        raise ValueError(f"image size {H}x{W} is not a positive multiple of {multiple}")


class AutoencoderKL(PackedModule):
    def __init__(self, ddconfig, embed_dim, scale_factor=1):
        super().__init__()
        self.encoder = Encoder(**ddconfig)
        self.decoder = Decoder(**ddconfig)
        assert ddconfig["double_z"]
        self.quant_conv = torch.nn.Conv2d(2 * ddconfig["z_channels"], 2 * embed_dim, 1)
        self.post_quant_conv = torch.nn.Conv2d(embed_dim, ddconfig["z_channels"], 1)
        self.embed_dim = embed_dim
        self.scale_factor = scale_factor

    def _pack(self):
        zc = self.post_quant_conv.out_channels
        mc = self.quant_conv.out_channels
        return {"wpq": f32(self.post_quant_conv.weight).reshape(zc, self.embed_dim).contiguous(),
                "bpq": f32(self.post_quant_conv.bias),
                "wq": f32(self.quant_conv.weight).reshape(mc, self.quant_conv.in_channels).contiguous(),
                "bq": f32(self.quant_conv.bias)}

    @torch.no_grad()
    def encode(self, x):
        """autoencoder.py:27-31.  Not on the sampling path from noise; its latent can start image-to-image sampling
        (the samplers' and `Request`'s `x_init`)."""
        h = self.encoder(x)
        moments = torch.nn.functional.conv2d(h, self.quant_conv.weight.float(), self.quant_conv.bias.float())
        return DiagonalGaussianDistribution(moments).sample() * self.scale_factor

    @torch.no_grad()
    def encode_images(self, images, seed=None):
        """uint8 RGB images (B, H, W, 3) -> fp32 latents (B, 4, H/8, W/8) on the model's device: `encode` of the images
        normalised as the reference's data loader does (u / 127.5 - 1 as NCHW, dataset/decode_item.py:567-568), that is
        posterior.sample() * scale_factor, with image b's posterior noise keyed by (seed, b) (include/idiff_b200.h
        idiff_encode_posterior).  So the latent of an image depends on the image, the seed and b alone, not on what else
        is encoded with it or before it.  seed: an integer in [0, 2^64), or None for one draw from torch's default CPU
        generator (`resolve_seed`)."""
        seed = resolve_seed(True, seed)
        return self._encode_images(images, [seed] * int(images.shape[0]), list(range(int(images.shape[0]))))

    def _encode_images(self, images, seeds, index):
        """`encode_images` with a seed and an in-request index per image, so one forward serves the images of many
        requests (batched.encode_images)."""
        if self.embed_dim != 4 or self.quant_conv.in_channels != 8:
            raise NotImplementedError("encode_images supports the shipped 4-channel latent (embed_dim 4, double_z)")
        check_images(images, 2 ** (self.encoder.num_resolutions - 1))
        p = self.pk()
        dev = p["wq"].device
        h = self.encoder.forward_images(images.to(dev).contiguous())
        index = torch.tensor([int(i) for i in index], dtype=torch.int32).to(dev)
        return ops.encode_posterior(h, p["wq"], p["bq"], float(self.scale_factor), ops.seed_array(seeds, dev), index)

    @torch.no_grad()
    def decode(self, z):
        """autoencoder.py:33-37: z (B, 4, h, w) -> image (B, 3, 8h, 8w) fp32 in [-1, 1] (nominally)."""
        if self.embed_dim != self.post_quant_conv.out_channels:
            raise NotImplementedError("post_quant_conv with embed_dim != z_channels is not used by the shipped configs")
        p = self.pk()
        B, _, H, W = z.shape
        z16 = ops.vae_latent_in(z.float().contiguous(), p["wpq"], p["bpq"], 1.0 / float(self.scale_factor))
        return self.decoder._decode_tokens(z16, B, H, W)

    @torch.no_grad()
    def decode_images(self, z):
        """z (B, 4, h, w) -> uint8 (B, 8h, 8w, 3) on the device: `decode(z)` and the bytes inference.py:122-125 saves
        (clamp to [-1, 1], * 0.5 + 0.5, * 255, truncated like astype(np.uint8)) in one kernel."""
        x = self.decode(z)
        B, _, H, W = x.shape
        return ops.decode_to_image(x, torch.empty((B, H, W, 3), dtype=torch.uint8, device=x.device))
