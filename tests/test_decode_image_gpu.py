"""`-m gpu` tests of the image output: the decode_to_image kernel against the reference's torch / numpy post-processing
(inference.py:122-125) in both storage builds, `AutoencoderKL.decode_images` on the latents of tests/golden/vae.pt,
image requests of `sample_requests` and `SamplingEngine` against each request's own sampler + `decode_images`, and
batch-invariant mode through the first stage."""
import math
import os
import sys
from dataclasses import replace

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import cases  # noqa: E402
import cases_decode as CDec  # noqa: E402
from test_ddim_gpu import DDIM_LATENT_TOL, _rel, diffusion, unet  # noqa: E402,F401 (module fixtures)
from test_engine_gpu import _drive  # noqa: E402
from test_img2img_gpu import _alone, _requests  # noqa: E402
from test_requests_gpu import _fresh, _reset  # noqa: E402

pytestmark = pytest.mark.gpu
DTYPES = [torch.float16, torch.bfloat16]
GOLDEN = os.path.join(HERE, "golden")


@pytest.fixture(scope="module")
def vae(cuda_device):
    from oracle import torch_oracle as TO
    from instancediffusion_b200.ldm.models.autoencoder import AutoencoderKL
    from instancediffusion_b200.weights import synth_tensor
    with torch.device("meta"):
        m = AutoencoderKL(dict(TO.VAE_DDCONFIG), 4, TO.VAE_SCALE)
    m = m.to_empty(device=cuda_device).eval()
    m.load_state_dict({k: synth_tensor("vae." + k, tuple(v.shape), cases.WEIGHT_SEED) for k, v in m.state_dict().items()},
                      strict=True)
    return m


def _compare(got: torch.Tensor, x: torch.Tensor, what: str, max_near: float = 1e-3) -> int:
    """The kernel's bytes against the reference's post-processing of x (fp32 NCHW): equal, or off by one where the fp32
    product (clamp(x) * 0.5 + 0.5) * 255 lies within one ulp of an integer, which may go either way; returns the number
    of such bytes and bounds them to `max_near` of all.  Measured on an H100: none in any case here (the kernel's fma
    rounds like the reference's mul + add, since x * 0.5 is exact)."""
    want = CDec.reference_post(x)
    got = got.cpu().numpy()
    assert got.dtype == np.uint8 and got.shape == want.shape, (got.shape, want.shape)
    xs = np.clip(x.cpu().numpy().transpose(0, 2, 3, 1), -1, 1)
    v = (xs * np.float32(0.5) + np.float32(0.5)) * np.float32(255)
    near = np.abs(v - np.round(v)) <= np.spacing(np.abs(v).astype(np.float32))
    diff = np.abs(got.astype(np.int32) - want.astype(np.int32))
    off = diff != 0
    n_off = int(off.sum())
    print(f"[{what}] {got.size} bytes, {n_off} off by one (all within 1 ulp of an integer), "
          f"{int(near.sum())} products within 1 ulp of an integer, {float((v == 0).mean() + (v == 255).mean()):.3f} "
          "clamped or at the ends")
    assert diff.max() <= 1, diff.max()
    assert not (off & ~near).any()
    assert n_off <= max_near * got.size, n_off
    return n_off


# ------------------------------------------------------------------------------------------------
# 1. the kernel
# ------------------------------------------------------------------------------------------------
def _decoder_like(shape, seed, device):
    """A random decoder output: mostly inside [-1, 1], a tenth of it beyond, and +-inf, -1, 1 and the values whose
    products sit at the byte boundaries."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(shape, generator=g) * 0.6
    flat = x.view(-1)
    k = torch.randint(0, 256, (flat.numel() // 8,), generator=g)
    idx = torch.randperm(flat.numel(), generator=g)[: k.numel()]
    flat[idx] = (2 * k.double() / 255 - 1).float()  # boundaries k/255, rounded to fp32 either side
    specials = torch.tensor([float("inf"), float("-inf"), -1.0, 1.0, 0.0, 3.0, -2.5])
    flat[: min(specials.numel(), flat.numel())] = specials[: flat.numel()]
    return x.to(device)


@pytest.mark.parametrize("build", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("in_dtype", ["fp32", "storage"])
@pytest.mark.parametrize("shape", [(2, 3, 64, 64), (1, 3, 512, 512), (3, 3, 5, 7), (1, 3, 1, 6)])
def test_decode_to_image_against_reference_post(cuda_device, build, in_dtype, shape):
    """(5, 7) and (1, 6): hw % 4 != 0, the element-by-element path."""
    from instancediffusion_b200 import ops
    with ops.storage(build):
        x = _decoder_like(shape, 11 + shape[0] * shape[2], cuda_device)
        if in_dtype == "storage":
            x = x.to(build)
        B, _, H, W = shape
        out = ops.decode_to_image(x, torch.full((B, H, W, 3), 77, dtype=torch.uint8, device=cuda_device))
        torch.cuda.synchronize()
    _compare(out, x.float(), f"decode_to_image {build} {in_dtype} {shape}")


def test_decode_to_image_nan_and_misaligned_input(cuda_device):
    """NaN gives 0 (the reference's astype of NaN is undefined); an input not 16-byte aligned takes the scalar path."""
    from instancediffusion_b200 import ops
    x = torch.full((1, 3, 2, 4), float("nan"), device=cuda_device)
    out = ops.decode_to_image(x, torch.full((1, 2, 4, 3), 9, dtype=torch.uint8, device=cuda_device))
    assert (out == 0).all()
    buf = _decoder_like((1, 3 * 64 * 64 + 1), 5, cuda_device).view(-1)
    x = buf[1:].view(1, 3, 64, 64)  # contiguous, 4 bytes past a 16-byte boundary
    assert x.data_ptr() % 16 == 4
    out = ops.decode_to_image(x, torch.empty((1, 64, 64, 3), dtype=torch.uint8, device=cuda_device))
    _compare(out, x, "decode_to_image misaligned")


def test_decode_to_image_rejects_bad_arguments(cuda_device):
    from instancediffusion_b200 import ops
    from instancediffusion_b200._lib import IdiffError
    x = torch.zeros((1, 3, 8, 8), device=cuda_device)
    out = torch.empty((1, 8, 8, 3), dtype=torch.uint8, device=cuda_device)
    bad = [
        (x.double(), out), (x.to(torch.bfloat16 if ops.storage_dtype() == torch.float16 else torch.float16), out),
        (torch.zeros((1, 4, 8, 8), device=cuda_device), out), (x[..., :4], out[:, :, :4]),
        (x, out.float()), (x, torch.empty((1, 8, 8, 4), dtype=torch.uint8, device=cuda_device)),
        (x, out.permute(0, 2, 1, 3)), (x.cpu(), out), (x.view(1, 3, 64), out),
    ]
    for a, b in bad:
        with pytest.raises(IdiffError):
            ops.decode_to_image(a, b)


# ------------------------------------------------------------------------------------------------
# 2. AutoencoderKL.decode_images
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", [n for n, s in cases.VAE_CASES.items() if s["kind"] == "decode"])
def test_decode_images_on_golden_latents(cuda_device, vae, name):
    """decode_images against decode + the reference's post-processing (the same decoder output: the kernel alone), and
    against the reference's post-processing of the reference's own fp32 image (the golden): there the bytes differ by
    the decoder's fp16 error, which test_vae_gpu bounds by 3e-3 of the image's largest magnitude."""
    spec = cases.VAE_CASES[name]
    g = torch.Generator().manual_seed(spec["seed"])
    z = (torch.randn((spec["batch"], 4, spec["size"], spec["size"]), generator=g) * spec["std"]).to(cuda_device)
    img = vae.decode_images(z)
    assert img.dtype == torch.uint8 and img.device == z.device
    assert img.shape == (spec["batch"], 8 * spec["size"], 8 * spec["size"], 3)
    _compare(img, vae.decode(z), f"decode_images {name}")
    path = os.path.join(GOLDEN, "vae.pt")
    if not os.path.exists(path):
        pytest.skip("vae.pt not generated")
    ref = torch.load(path, map_location="cpu")[name].float()
    want = CDec.reference_post(ref)
    diff = np.abs(img.cpu().numpy().astype(np.int32) - want.astype(np.int32))
    bound = math.ceil(3e-3 * ref.abs().max().item() * 127.5) + 1  # +1: truncation may cross a boundary
    print(f"[decode_images {name} vs golden] max byte diff {diff.max()} (bound {bound}), mean {diff.mean():.4f}, "
          f"{(diff != 0).mean():.4f} of bytes differ")
    assert diff.max() <= bound


# ------------------------------------------------------------------------------------------------
# 3. the request drivers
# ------------------------------------------------------------------------------------------------
OUTPUTS = ["image", "image", "latent", "image", "latent", "image"]  # over test_img2img_gpu._requests


def _image_rel(a: torch.Tensor, b: torch.Tensor) -> float:
    """Relative L2 of two uint8 images as values in [-1, 1]."""
    return _rel(a.double() / 127.5 - 1, b.double() / 127.5 - 1)


def _check_outputs(got, reqs, alone_latents, vae, what):
    for k, (r, lat) in enumerate(zip(reqs, alone_latents)):
        if r.output == "latent":
            rel = _rel(got[k], lat)
        else:
            want = vae.decode_images(lat)
            assert got[k].dtype == torch.uint8 and got[k].shape == want.shape, (k, got[k].shape)
            rel = _image_rel(got[k], want)
        print(f"[{what}] request {k} ({r.sampler}, strength {r.strength}, {r.output}): rel_l2 vs alone {rel:.2e}")
        # an image inherits the latents' difference (the forwards' rounding, DDIM_LATENT_TOL) through the decoder
        assert rel < (DDIM_LATENT_TOL if r.output == "latent" else 2 * DDIM_LATENT_TOL), (k, rel)


def test_sample_requests_images_match_each_request_alone(cuda_device, unet, diffusion, vae):
    from instancediffusion_b200.ldm.models.diffusion.batched import sample_requests
    reqs = [replace(r, output=o) for r, o in zip(_requests(unet, cuda_device), OUTPUTS)]
    alone = [_alone(unet, diffusion, r) for r in reqs]
    _reset(unet)
    try:
        got = sample_requests(unet, diffusion, [_fresh(r) for r in reqs], 10, max_batch=8, autoencoder=vae,
                              max_decode_batch=3)
    finally:
        _reset(unet)
    _check_outputs(got, reqs, alone, vae, "sample_requests images")


def test_engine_images_match_each_request_alone(cuda_device, unet, diffusion, vae):
    from instancediffusion_b200.ldm.models.diffusion.engine import SamplingEngine
    reqs = [replace(r, output=o) for r, o in zip(_requests(unet, cuda_device), OUTPUTS)]
    reqs[1], reqs[4] = replace(reqs[1], S=11), replace(reqs[4], S=11)
    alone = [_alone(unet, diffusion, r) for r in reqs]
    _reset(unet)
    try:
        got = _drive(SamplingEngine(unet, diffusion, max_batch=8, autoencoder=vae), reqs, [0, 0, 2, 3, 5, 6])
    finally:
        _reset(unet)
    _check_outputs(got, reqs, alone, vae, "engine images")


# ------------------------------------------------------------------------------------------------
# 4. batch-invariant mode through the first stage
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=["fp16", "bf16"])
def test_batch_invariant_decode(cuda_device, vae, dtype):
    """With the mode on, every decoder kernel (GEMM / conv3x3, GroupNorm, the mid-block attention's per-image scores,
    softmax and P V, the latent prologue, the upsampling and the image epilogue) gives an image the same bytes at any
    decode batch."""
    from instancediffusion_b200 import ops
    g = torch.Generator().manual_seed(21)
    z = (torch.randn((5, 4, 64, 64), generator=g) * 0.9).to(cuda_device)
    with ops.storage(dtype):
        ops.set_batch_invariant(True)
        try:
            together = vae.decode_images(z)
            for j in range(5):
                assert torch.equal(vae.decode_images(z[j:j + 1]), together[j:j + 1]), j
            assert torch.equal(vae.decode_images(z[1:4]), together[1:4])
        finally:
            ops.set_batch_invariant(False)


@pytest.mark.parametrize("dtype", DTYPES, ids=["fp16", "bf16"])
def test_batch_invariant_image_requests(cuda_device, unet, diffusion, vae, dtype):
    """With the mode on, an image request's bytes are the same alone (its own sampler + decode_images), in
    sample_requests and in SamplingEngine, however the requests and their decodes are batched."""
    from instancediffusion_b200 import ops
    from instancediffusion_b200.ldm.models.diffusion.batched import sample_requests
    from instancediffusion_b200.ldm.models.diffusion.engine import SamplingEngine
    with ops.storage(dtype):
        ops.set_batch_invariant(True)
        try:
            reqs = [replace(r, output=o) for r, o in zip(_requests(unet, cuda_device), OUTPUTS)]
            targets = (0, 1, 5)
            alone = {j: vae.decode_images(_alone(unet, diffusion, reqs[j])) for j in targets}
            got = sample_requests(unet, diffusion, [_fresh(r) for r in reqs], 10, max_batch=8, autoencoder=vae,
                                  max_decode_batch=2)
            _reset(unet)
            for j in targets:
                assert torch.equal(got[j], alone[j]), j
            got = _drive(SamplingEngine(unet, diffusion, max_batch=8, buckets=(2, 4, 8), autoencoder=vae),
                         reqs, [0, 1, 0, 2, 0, 3])
            _reset(unet)
            for j in targets:
                assert torch.equal(got[j], alone[j]), j
        finally:
            ops.set_batch_invariant(False)
            _reset(unet)
