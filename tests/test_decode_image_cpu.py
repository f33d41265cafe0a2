"""`output="image"` without a GPU: the request validation, the missing-autoencoder errors, the torch restatement of the
decode_to_image kernel against numpy's astype(np.uint8) at the edges, and image requests next to latent ones in
`sample_requests` and `SamplingEngine` on the fake UNet with a fake first stage (tests/cases_decode.py)."""
import os
import sys
from dataclasses import replace

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import cases_decode as CDec  # noqa: E402
from fake_unet import FakeUNet, _fresh, _req, torch_kernels  # noqa: E402,F401
from instancediffusion_b200.ldm.models.diffusion.batched import (  # noqa: E402
    RequestPlan, check_requests, decode_latents, sample_requests)
from instancediffusion_b200.ldm.models.diffusion.engine import SamplingEngine  # noqa: E402


@pytest.fixture
def diffusion():
    from instancediffusion_b200.ldm.models.diffusion.ldm import LatentDiffusion
    return LatentDiffusion(linear_start=0.00085, linear_end=0.012, timesteps=1000)


# ------------------------------------------------------------------------------------------------
# validation
# ------------------------------------------------------------------------------------------------
def test_check_requests_output(diffusion):
    ok = _req(1, 10)
    assert check_requests([replace(ok, output="image"), ok], 10, 32) == [RequestPlan(1, None, 1, True, 0)] * 2
    for bad in ("images", "Image", "png", None):
        with pytest.raises(ValueError, match=r"request 1: unknown output"):
            check_requests([ok, replace(ok, output=bad)], 10, 32)


def test_missing_autoencoder_raises(diffusion, torch_kernels):
    model = FakeUNet()
    img = replace(_req(2, 10), output="image")
    with pytest.raises(ValueError, match="request 1: output='image' needs the driver's autoencoder"):
        sample_requests(model, diffusion, [_req(3, 10), img], 10)
    assert model.calls == []  # raised at entry, before any forward
    with pytest.raises(ValueError, match="max_decode_batch"):
        sample_requests(model, diffusion, [img], 10, autoencoder=CDec.FakeAutoencoder(), max_decode_batch=0)
    eng = SamplingEngine(model, diffusion)
    with pytest.raises(ValueError, match="needs the driver's autoencoder"):
        eng.submit(img)
    assert eng.queued == []
    with pytest.raises(ValueError, match="max_decode_batch"):
        SamplingEngine(model, diffusion, autoencoder=CDec.FakeAutoencoder(), max_decode_batch=-1)


# ------------------------------------------------------------------------------------------------
# the restated kernel against numpy
# ------------------------------------------------------------------------------------------------
def _edges() -> np.ndarray:
    """-1, 1, 0, +-inf, out-of-range values, and for every byte boundary k/255 the fp32 inputs whose product
    (x * 0.5 + 0.5) * 255 lands just below, at and just above k, with their fp32 neighbours."""
    xs = [-1.0, 1.0, 0.0, -0.0, np.inf, -np.inf, 2.0, -3.5, 1e30, -1e30, np.nextafter(np.float32(1), np.float32(0)),
          np.nextafter(np.float32(-1), np.float32(0))]
    for k in range(256):
        x = np.float32(2 * k / 255 - 1)
        for _ in range(4):  # walk down to the fp32 inputs just below the boundary
            xs.append(x)
            x = np.nextafter(x, np.float32(-2))
        x = np.float32(2 * k / 255 - 1)
        for _ in range(4):
            x = np.nextafter(x, np.float32(2))
            xs.append(x)
    return np.array(xs, dtype=np.float32)


def test_restated_truncation_matches_numpy():
    xs = _edges()
    t = torch.from_numpy(xs).view(1, 1, 1, -1).expand(1, 3, 1, -1).contiguous()
    got = CDec.restated_post(t).numpy()
    with np.errstate(invalid="ignore"):
        want = CDec.reference_post(t)
    assert got.shape == want.shape == (1, 1, xs.size, 3)
    assert np.array_equal(got, want)
    got = got[0, 0, :, 0]
    assert got[0] == 0 and got[1] == 255 and got[4] == 255 and got[5] == 0  # -1, 1, +inf, -inf
    assert got[2] == 127  # (0 * 0.5 + 0.5) * 255 = 127.5 truncates
    # the byte boundaries are truncated, not rounded: somewhere below k/255 the byte is k - 1
    v = (np.clip(xs, -1, 1) * np.float32(0.5) + np.float32(0.5)) * np.float32(255)
    below = (v < np.round(v)) & (np.round(v) - v < 1e-3)
    assert below.any() and np.array_equal(got[below], np.round(v[below]).astype(np.uint8) - 1)


def test_restated_post_on_random_decoder_outputs():
    x = torch.randn((2, 3, 16, 24), generator=torch.Generator().manual_seed(3)) * 1.3
    assert np.array_equal(CDec.restated_post(x).numpy(), CDec.reference_post(x))


# ------------------------------------------------------------------------------------------------
# the request drivers
# ------------------------------------------------------------------------------------------------
def _batch2(req):
    """The request at batch 2 (two images of one layout)."""
    g = torch.Generator().manual_seed(77)
    return replace(req, input=dict(req.input, x=torch.randn((2, 4, 64, 64), generator=g),
                                   context=req.input["context"].expand(2, -1, -1)))


def _mix(S):
    """Plain PLMS, DDIM at eta 0.7, Multi-instance, image-to-image and batch-2 requests."""
    return [
        _req(80, S),
        replace(_req(81, S), sampler="ddim", eta=0.7, seed=1234),
        _req(82, S, n=2, mis=0.36),
        replace(_req(83, S), x_init=torch.randn((1, 4, 64, 64), generator=torch.Generator().manual_seed(5)),
                strength=0.6, seed=21),
        _batch2(_req(84, S)),
        replace(_req(85, S), sampler="ddim"),
    ]


@pytest.mark.parametrize("max_decode_batch", [8, 2])
def test_sample_requests_mixes_image_and_latent_requests(diffusion, torch_kernels, max_decode_batch):
    S = 10
    reqs = _mix(S)
    latents = sample_requests(FakeUNet(scale=0.5), diffusion, [_fresh(r) for r in reqs], S, max_batch=8)
    out_kind = ["image", "latent", "image", "image", "image", "latent"]
    vae = CDec.FakeAutoencoder()
    got = sample_requests(FakeUNet(scale=0.5), diffusion, [replace(_fresh(r), output=o) for r, o in zip(reqs, out_kind)],
                          S, max_batch=8, autoencoder=vae, max_decode_batch=max_decode_batch)
    for k, (o, lat) in enumerate(zip(out_kind, latents)):
        if o == "latent":
            assert torch.equal(got[k], lat), k  # bit-for-bit what a latent-only run gives
        else:
            want = CDec.restated_post(CDec.fake_decode(lat))
            assert got[k].dtype == torch.uint8 and got[k].shape == (lat.shape[0], 512, 512, 3), k
            assert torch.equal(got[k], want), k
    images = 1 + 1 + 1 + 2  # the batch-2 request decodes both its images
    assert sum(vae.calls) == images and max(vae.calls) <= max_decode_batch
    assert len(vae.calls) == -(-images // max_decode_batch)  # decoded together, in as few chunks as the bound allows


def test_sample_requests_latent_only_ignores_the_autoencoder(diffusion, torch_kernels):
    reqs = _mix(10)
    a = sample_requests(FakeUNet(), diffusion, [_fresh(r) for r in reqs], 10, max_batch=8)
    vae = CDec.FakeAutoencoder()
    b = sample_requests(FakeUNet(), diffusion, [_fresh(r) for r in reqs], 10, max_batch=8, autoencoder=vae)
    assert vae.calls == [] and all(torch.equal(x, y) for x, y in zip(a, b))


@pytest.mark.parametrize("max_decode_batch", [8, 3])
def test_engine_decodes_a_tick_together(diffusion, torch_kernels, max_decode_batch):
    """Five image requests (six images) finish in the same tick and are decoded in that tick, in chunks of at most
    max_decode_batch images; two latent requests finishing with them and one image request finishing later are
    unaffected."""
    S = 10
    base = [replace(_req(90 + k, S), output="image") for k in range(4)] + [replace(_batch2(_req(95, S)), output="image")]
    latent = [_req(96, S), replace(_req(97, S), sampler="ddim", eta=0.5, seed=3)]
    late = replace(_req(98, S), output="image")
    vae = CDec.FakeAutoencoder()
    eng = SamplingEngine(FakeUNet(), diffusion, max_batch=8, buckets=None, autoencoder=vae,
                         max_decode_batch=max_decode_batch)
    tickets = [eng.submit(_fresh(r)) for r in base + [latent[0]]]
    eng.step()  # the DDIM request retires a tick before the PLMS ones: submitting it a tick later aligns them
    tickets.append(eng.submit(_fresh(latent[1])))
    out, finished_at, tick = {}, {}, 1
    while eng.queued or eng.live:
        if tick == 3:
            tickets.append(eng.submit(_fresh(late)))
        calls = len(vae.calls)
        for t, x in eng.step().items():
            out[t], finished_at[t] = x, tick
        if len(vae.calls) > calls:
            decoded = vae.calls[calls:]
            if tick == finished_at[tickets[0]]:
                assert sum(decoded) == 6 and max(decoded) <= max_decode_batch
                assert len(decoded) == -(-6 // max_decode_batch), decoded
            else:
                assert decoded == [1]
        tick += 1
    assert len({finished_at[t] for t in tickets[:7]}) == 1
    assert finished_at[tickets[7]] > finished_at[tickets[0]]
    # each request against its latent from a latent-only engine run
    plain = SamplingEngine(FakeUNet(), diffusion, max_batch=8, buckets=None)
    pt = [plain.submit(_fresh(replace(r, output="latent"))) for r in base + [latent[0]]]
    plain.step()
    pt.append(plain.submit(_fresh(latent[1])))
    lat = dict(plain.step())
    while plain.queued or plain.live:
        lat.update(plain.step())
    for t, p in zip(tickets[:5], pt[:5]):
        assert torch.equal(out[t], CDec.restated_post(CDec.fake_decode(lat[p])))
    for t, p in zip(tickets[5:7], pt[5:7]):
        assert torch.equal(out[t], lat[p])
    assert out[tickets[4]].shape == (2, 512, 512, 3)


def test_decode_latents_groups_by_size(torch_kernels):
    vae = CDec.FakeAutoencoder()
    g = torch.Generator().manual_seed(9)
    zs = [torch.randn(s, generator=g) for s in ((1, 4, 8, 8), (2, 4, 4, 8), (3, 4, 8, 8), (1, 4, 4, 8))]
    got = decode_latents(vae, zs, 3)
    assert sorted(vae.calls) == [1, 3, 3]  # 4 images of 8x8 in chunks of 3 and 1, 3 of 4x8 in one
    for z, img in zip(zs, got):
        assert torch.equal(img, CDec.restated_post(CDec.fake_decode(z)))
