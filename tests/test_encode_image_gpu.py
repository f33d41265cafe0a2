"""`-m gpu` tests of image-to-image from images: the image-in conv kernel against torch's fp32 conv of u / 127.5 - 1 and
against the padded-copy + conv GEMM path it replaces, the posterior kernel against its float64 restatement, and
`AutoencoderKL.encode_images` against the plain-torch restatement of the reference encoder, in both storage builds;
batch invariance of the encode, and `init_image` requests next to latent, x_init, DDIM, DPM-Solver++(2M) and image
requests in `sample_requests` and `SamplingEngine` against the same requests given x_init = encode_images(...)."""
import os
import sys
from dataclasses import replace

import numpy as np
import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import cases_encode as CE  # noqa: E402
from test_ddim_gpu import DDIM_LATENT_TOL, _rel, diffusion, unet  # noqa: E402,F401 (module fixtures)
from test_decode_image_gpu import _image_rel, vae  # noqa: E402,F401 (module fixture)
from test_engine_gpu import _drive  # noqa: E402
from test_img2img_gpu import _requests  # noqa: E402
from test_requests_gpu import _fresh, _reset  # noqa: E402

pytestmark = pytest.mark.gpu
DTYPES = [torch.float16, torch.bfloat16]
UNIT = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}  # unit roundoff of the storage type
# relative L2 of encode_images against the fp32 restatement, about 2x the value measured on an H100
ENCODE_TOL = {torch.float16: 1.4e-3, torch.bfloat16: 1.1e-2}  # measured 6.8e-4 / 5.3e-3


class _fp32_torch:
    """torch's convolutions and matmuls in plain fp32 (no TF32) inside the block."""

    def __enter__(self):
        self.prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False

    def __exit__(self, *exc):
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = self.prev


def _normalised(images: torch.Tensor) -> torch.Tensor:
    """The reference data loader's image: arr.astype(np.float32) / 127.5 - 1, NCHW (dataset/decode_item.py:567-568)."""
    return (images.float() / 127.5 - 1).permute(0, 3, 1, 2).contiguous()


# ------------------------------------------------------------------------------------------------
# 1. the kernels
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("H,W,batch", [(64, 64, 1), (64, 64, 3), (512, 512, 1), (512, 512, 3), (40, 200, 2)])
def test_image_in_against_fp32_conv_and_the_padded_path(cuda_device, vae, dtype, H, W, batch):
    """Each output within 2u|y| (the storage type's rounding of the output: one ulp) + u S (the weights rounded to
    the storage type) + 1e-6 S (fp32 summation of 27 terms), S = sum |w| |x|; the padded path (image rounded to the
    storage type, conv GEMM) within the same bound plus u S for its rounded input.  40 x 200 splits rows into a full
    and a partial segment."""
    from instancediffusion_b200 import ops
    images = CE.random_images(batch, H, W, 100 + H + batch).to(cuda_device)
    conv = vae.encoder.conv_in
    with ops.storage(dtype):
        p = vae.encoder.pk()
        got = ops.encode_image_in(images, p["w_img"], p["b_in"]).float()
        x = _normalised(images)
        B = batch
        padded = ops.gemm(ops.nchw_f32_to_nhwc_f16(x, 64), p["w_in"], p["b_in"], conv=(B, H, W, 64)).float()
    with _fp32_torch(), torch.no_grad():
        ref = F.conv2d(x, conv.weight.float(), conv.bias.float(), padding=1).permute(0, 2, 3, 1).reshape(-1, 128)
        s = F.conv2d(x.abs(), conv.weight.float().abs(), padding=1).permute(0, 2, 3, 1).reshape(-1, 128)
    u = UNIT[dtype]
    bound = 2 * u * ref.abs() + u * s + 1e-6 * s + 1e-30
    err, err_pad = (got - ref).abs(), (padded - ref).abs()
    print(f"[image_in {dtype} {batch}x{H}x{W}] max err/bound {float((err / bound).max()):.3f}, padded path "
          f"{float((err_pad / (bound + u * s)).max()):.3f}; rel L2 {float((got - ref).norm() / ref.norm()):.2e}, padded "
          f"{float((padded - ref).norm() / ref.norm()):.2e}")
    assert bool((err <= bound).all())
    assert bool((err_pad <= bound + u * s).all())
    assert bool(((got - padded).abs() <= 2 * bound + u * s).all())


@pytest.mark.parametrize("hw", [(8, 8), (3, 5), (64, 64)])
def test_posterior_against_float64(cuda_device, hw):
    """The kernel against (mean + exp(0.5 clamp(logvar)) eps) * scale in float64 with the restated noise stream:
    per element within 1e-5 of the terms' magnitudes.  Odd sizes split a noise group across channels; seeds above 2^63
    and nonzero indices exercise the key and counter words; logvars reach past both clamps."""
    from instancediffusion_b200 import ops
    g = torch.Generator().manual_seed(31 + hw[0])
    B = 4
    h = (torch.randn((B, 8, *hw), generator=g) * 3).to(cuda_device)
    h[:, 7] = torch.linspace(-80, 60, hw[0] * hw[1]).view(hw)  # through the bias-free last row below: past the clamps
    w = (torch.randn((8, 8), generator=g) * 0.3)
    w[7] = 0
    w[7, 7] = 1
    w = w.to(cuda_device)
    b = (torch.randn((8,), generator=g) * 0.1).to(cuda_device)
    b[7] = 0
    seeds, index = [5, 2 ** 64 - 1, 2 ** 63 + 7, 5], [0, 1, 3, 2]
    z = ops.encode_posterior(h, w, b, CE.SCALE, ops.seed_array(seeds, cuda_device),
                             torch.tensor(index, dtype=torch.int32, device=cuda_device))
    m = CE.quant_conv64(h, w, b).cpu()
    want = CE.posterior(m, CE.SCALE, seeds, index)
    # the terms' magnitudes: the quant_conv sum of the mean, and std (|eps| + 1) since eps is fp32 Box-Muller
    std = torch.exp(0.5 * m[:, 4:].clamp(-30, 20))
    mag = CE.SCALE * (torch.einsum("ok,bkhw->bohw", w.double().abs().cpu(), h.double().abs().cpu())[:, :4]
                      + b.double().abs().cpu().view(1, 8, 1, 1)[:, :4] + (want / CE.SCALE - m[:, :4]).abs() + std)
    err = (z.double().cpu() - want).abs()
    print(f"[posterior {hw}] max err/magnitude {float((err / mag).max()):.2e}")
    assert bool((err <= 1e-5 * mag).all())


def test_kernels_reject_bad_arguments(cuda_device, vae):
    from instancediffusion_b200 import _lib, ops
    p = vae.encoder.pk()
    img = CE.random_images(1, 16, 16, 1).to(cuda_device)
    for bad in (img.float(), img[..., :2].contiguous(), img.cpu(), img.permute(0, 2, 1, 3)):
        with pytest.raises(_lib.IdiffError):
            ops.encode_image_in(bad, p["w_img"], p["b_in"])
    with pytest.raises(_lib.IdiffError):
        ops.encode_image_in(img, p["w_in"], p["b_in"])
    h = torch.zeros((2, 8, 4, 4), device=cuda_device)
    w, b = torch.zeros((8, 8), device=cuda_device), torch.zeros((8,), device=cuda_device)
    s, i = ops.seed_array([1, 2], cuda_device), torch.zeros((2,), dtype=torch.int32, device=cuda_device)
    for args in ((h[:, :4].contiguous(), w, b, 1.0, s, i), (h, w, b, 1.0, s[:1], i), (h, w, b, 1.0, s, i.long()),
                 (h, w[:4], b, 1.0, s, i), (h.half(), w, b, 1.0, s, i)):
        with pytest.raises(_lib.IdiffError):
            ops.encode_posterior(*args)
    with pytest.raises(_lib.IdiffError):
        ops.seed_array([2 ** 64], cuda_device)


# ------------------------------------------------------------------------------------------------
# 2. AutoencoderKL.encode_images
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("size,batch", [(64, 2), (512, 1)])
def test_encode_images_against_fp32_restatement(cuda_device, vae, dtype, size, batch):
    """encode_images against oracle.torch_oracle.vae_encode_moments (the reference encoder in plain fp32 torch) and the
    restated posterior with the same seed: relative L2 of the latent."""
    from oracle import torch_oracle as TO
    from instancediffusion_b200 import ops
    images = CE.random_images(batch, size, size, 7 + size).to(cuda_device)
    seed = 2 ** 63 + 12345
    with ops.storage(dtype):
        z = vae.encode_images(images, seed=seed)
    sd = {k: v.detach().float() for k, v in vae.state_dict().items()}
    with _fp32_torch(), torch.no_grad():
        mom = TO.vae_encode_moments(sd, _normalised(images))
    want = CE.posterior(mom, TO.VAE_SCALE, [seed] * batch, list(range(batch)))
    assert z.shape == (batch, 4, size // 8, size // 8) and z.dtype == torch.float32
    rel = _rel(z, want)
    rel_mean = _rel(z, CE.posterior(mom, TO.VAE_SCALE, [seed + 1] * batch, list(range(batch))))
    print(f"[encode_images {dtype} {batch}x{size}] rel_l2 vs restated {rel:.3e} (another seed: {rel_mean:.3e})")
    assert rel < ENCODE_TOL[dtype], rel
    assert rel_mean > 10 * rel  # the noise is the seed's: another seed lands far away


def test_encode_images_seeding(cuda_device, vae):
    images = CE.random_images(2, 64, 64, 3).to(cuda_device)
    a = vae.encode_images(images, seed=9)
    assert torch.equal(a, vae.encode_images(images.cpu(), seed=9))  # moved to the model's device, same result
    torch.manual_seed(4)
    c = vae.encode_images(images)
    torch.manual_seed(4)
    assert torch.equal(c, vae.encode_images(images))  # seed=None: one draw from the default generator
    assert not torch.equal(c, a)
    with pytest.raises(ValueError):
        vae.encode_images(images.float())
    with pytest.raises(ValueError):
        vae.encode_images(images[:, :60])


@pytest.mark.parametrize("dtype", DTYPES, ids=["fp16", "bf16"])
def test_encode_images_batch_invariant(cuda_device, vae, dtype):
    """With batch-invariant mode on, an image's latent is bit-identical alone and inside a batch of 5 (the image-in
    conv, conv GEMMs, GroupNorm, im2col, per-image attention, the posterior)."""
    from instancediffusion_b200 import ops
    images = CE.random_images(5, 64, 64, 17).to(cuda_device)
    seeds, index = [3, 3, 8, 2 ** 64 - 2, 3], [0, 1, 0, 0, 2]
    with ops.storage(dtype):
        ops.set_batch_invariant(True)
        try:
            together = vae._encode_images(images, seeds, index)
            for j in range(5):
                assert torch.equal(vae._encode_images(images[j:j + 1], seeds[j:j + 1], index[j:j + 1]),
                                   together[j:j + 1]), j
            assert torch.equal(vae.encode_images(images[:2], seed=3), together[:2])
        finally:
            ops.set_batch_invariant(False)


# ------------------------------------------------------------------------------------------------
# 3. the request drivers
# ------------------------------------------------------------------------------------------------
def _mixed(unet, device, vae):
    """(init_image form, x_init form) of seven requests: image-to-image PLMS, DDIM at eta 0.7 (batch 2 from one image),
    and DPM-Solver++(2M) from images; a Multi-instance request from a latent; plain PLMS and DDIM; outputs mixed."""
    reqs = _requests(unet, device)
    imgs = {0: CE.random_images(1, 512, 512, 40), 1: CE.random_images(1, 512, 512, 41),
            5: CE.random_images(1, 512, 512, 42)}
    dpm = replace(reqs[4], sampler="dpmpp_2m", strength=0.5, seed=16)
    reqs = [reqs[0], reqs[1], reqs[2], reqs[4], reqs[5], dpm]
    outputs = ["image", "latent", "latent", "image", "latent", "image"]
    with_image, with_latent = [], []
    for j, (r, o) in enumerate(zip(reqs, outputs)):
        r = replace(r, output=o)
        if j in imgs:
            with_image.append(replace(r, x_init=None, init_image=imgs[j]))
            with_latent.append(replace(r, x_init=vae.encode_images(imgs[j], seed=r.seed), init_image=None))
        else:
            with_image.append(r)
            with_latent.append(r)
    return with_image, with_latent


def _compare(got, want, reqs, exact, what):
    for k, r in enumerate(reqs):
        if exact:
            assert torch.equal(got[k], want[k]), (what, k)
            continue
        rel = _rel(got[k], want[k]) if r.output == "latent" else _image_rel(got[k], want[k])
        print(f"[{what}] request {k} ({r.sampler}, {r.output}, init_image {r.init_image is not None}): "
              f"rel_l2 vs the x_init form {rel:.2e}")
        assert rel < (DDIM_LATENT_TOL if r.output == "latent" else 2 * DDIM_LATENT_TOL), (k, rel)


def _run_both(unet, diffusion, vae, device):
    from instancediffusion_b200.ldm.models.diffusion.batched import sample_requests
    from instancediffusion_b200.ldm.models.diffusion.engine import SamplingEngine
    with_image, with_latent = _mixed(unet, device, vae)
    out = {}
    try:
        for name, reqs in (("image", with_image), ("latent", with_latent)):
            _reset(unet)
            fresh = [_fresh(r) for r in reqs]
            a = sample_requests(unet, diffusion, fresh, 10, max_batch=8, autoencoder=vae, max_encode_batch=2)
            assert all(f.x_init is None for f in fresh if f.init_image is not None)  # the latent stays with the driver
            _reset(unet)
            b = _drive(SamplingEngine(unet, diffusion, max_batch=8, buckets=(2, 4, 8), autoencoder=vae,
                                      max_encode_batch=2), reqs, [0, 0, 1, 2, 2, 3])
            out[name] = (a, [b[j] for j in range(len(reqs))])
    finally:
        _reset(unet)
    return with_image, out


def test_init_image_requests_match_the_x_init_form(cuda_device, unet, diffusion, vae):
    reqs, out = _run_both(unet, diffusion, vae, cuda_device)
    _compare(out["image"][0], out["latent"][0], reqs, False, "sample_requests init_image")
    _compare(out["image"][1], out["latent"][1], reqs, False, "engine init_image")


@pytest.mark.parametrize("dtype", DTYPES, ids=["fp16", "bf16"])
def test_batch_invariant_init_image_requests(cuda_device, unet, diffusion, vae, dtype):
    """With the mode on, an init_image request gives the same bits as the same request with x_init =
    encode_images(init_image, seed=seed), in both drivers, whatever it is encoded and sampled with."""
    from instancediffusion_b200 import ops
    with ops.storage(dtype):
        ops.set_batch_invariant(True)
        try:
            reqs, out = _run_both(unet, diffusion, vae, cuda_device)
        finally:
            ops.set_batch_invariant(False)
    _compare(out["image"][0], out["latent"][0], reqs, True, "sample_requests init_image")
    _compare(out["image"][1], out["latent"][1], reqs, True, "engine init_image")


def test_image_output_refined_from_its_own_image(cuda_device, unet, diffusion, vae):
    """An output="image" result fed back as the next request's init_image (synthetic weights: the refined image is not
    expected to resemble its start)."""
    from instancediffusion_b200.ldm.models.diffusion.batched import sample_requests
    r = replace(_requests(unet, cuda_device)[4], output="image")
    try:
        _reset(unet)
        img = sample_requests(unet, diffusion, [_fresh(r)], 10, autoencoder=vae)[0]
        _reset(unet)
        again = sample_requests(unet, diffusion, [_fresh(replace(r, init_image=img, strength=0.3, seed=5))], 10,
                                autoencoder=vae)[0]
    finally:
        _reset(unet)
    assert img.shape == again.shape == (1, 512, 512, 3) and again.dtype == torch.uint8
    rel = _image_rel(again, img)
    print(f"[refine] image rel_l2 after strength 0.3: {rel:.3e}")
    assert rel > 0 and np.isfinite(rel)
