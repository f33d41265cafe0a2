"""`init_image` without a GPU: the request validation, the seed resolution order, how the drivers batch the encode, and
`init_image` requests against the same requests given x_init = encode_images(init_image, seed=seed) in
`sample_requests` and `SamplingEngine`, on the fake UNet with a fake first stage (tests/cases_encode.py)."""
import os
import sys
from dataclasses import replace

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import cases_encode as CE  # noqa: E402
from fake_unet import FakeUNet, _fresh, _req, torch_kernels  # noqa: E402,F401
from instancediffusion_b200.ldm.models.diffusion.batched import (  # noqa: E402
    RequestPlan, check_requests, encode_images, sample_requests)
from instancediffusion_b200.ldm.models.diffusion.engine import SamplingEngine  # noqa: E402


@pytest.fixture
def diffusion():
    from instancediffusion_b200.ldm.models.diffusion.ldm import LatentDiffusion
    return LatentDiffusion(linear_start=0.00085, linear_end=0.012, timesteps=1000)


def _img(seed, b=1, size=512):
    return CE.random_images(b, size, size, seed)


# ------------------------------------------------------------------------------------------------
# validation
# ------------------------------------------------------------------------------------------------
def test_check_requests_init_image():
    ok = _req(1, 10)
    assert check_requests([replace(ok, init_image=_img(1), strength=0.35)], 10, 32) == [RequestPlan(1, None, 1, True, 7)]
    assert check_requests([replace(ok, init_image=_img(1))], 10, 32) == [RequestPlan(1, None, 1, True, 0)]
    mis = replace(_req(3, 10, n=2, mis=0.36), init_image=_img(1), strength=0.35)
    assert check_requests([mis], 10, 32) == [RequestPlan(1, None, 1, True, 7)]  # merge before k0: global alone
    bad = [
        (_img(1).float(), "init_image must be a uint8 tensor"),
        (_img(1)[0], "does not fit the latent"),  # rank 3
        (_img(1, size=256), "does not fit the latent"),  # not 8x the 64x64 latent
        (_img(1)[:, :, :, :2], "does not fit the latent"),  # not RGB
        (_img(1, b=2), "does not fit the latent"),  # batch 2 on a batch-1 request
        (_img(1).permute(0, 3, 1, 2), "does not fit the latent"),  # NCHW
    ]
    for im, msg in bad:
        with pytest.raises(ValueError, match=f"request 1: (init_image of shape .* )?{msg}"):
            check_requests([ok, replace(ok, init_image=im, strength=0.5)], 10, 32)
    with pytest.raises(ValueError, match="request 0: x_init and init_image are exclusive"):
        check_requests([replace(ok, init_image=_img(1), x_init=torch.zeros((1, 4, 64, 64)), strength=0.5)], 10, 32)
    with pytest.raises(ValueError, match="request 0: strength=0.5 needs x_init or init_image"):
        check_requests([replace(ok, strength=0.5)], 10, 32)
    with pytest.raises(ValueError, match="request 0: strength=1.5 outside"):
        check_requests([replace(ok, init_image=_img(1), strength=1.5)], 10, 32)
    with pytest.raises(ValueError, match="inpainting"):  # still rejected with init_image
        check_requests([replace(ok, init_image=_img(1), mask=torch.zeros((1, 4, 64, 64)),
                                x0=torch.zeros((1, 4, 64, 64)))], 10, 32)


def test_missing_autoencoder_and_max_encode_batch(diffusion, torch_kernels):
    model = FakeUNet()
    req = replace(_req(2, 10), init_image=_img(2), strength=0.5, seed=1)
    with pytest.raises(ValueError, match="request 1: init_image needs the driver's autoencoder"):
        sample_requests(model, diffusion, [_req(3, 10), req], 10)
    assert model.calls == []  # raised at entry, before any forward
    for bad in (0, -2):
        with pytest.raises(ValueError, match="max_encode_batch must be positive"):
            sample_requests(model, diffusion, [req], 10, autoencoder=CE.FakeAutoencoder(), max_encode_batch=bad)
        with pytest.raises(ValueError, match="max_encode_batch must be positive"):
            SamplingEngine(model, diffusion, autoencoder=CE.FakeAutoencoder(), max_encode_batch=bad)
    eng = SamplingEngine(model, diffusion)
    with pytest.raises(ValueError, match="init_image needs the driver's autoencoder"):
        eng.submit(req)
    assert eng.queued == []


# ------------------------------------------------------------------------------------------------
# the seeds
# ------------------------------------------------------------------------------------------------
def test_encode_images_seed(torch_kernels):
    vae = CE.FakeAutoencoder()
    im = _img(4, b=2, size=64)
    a = vae.encode_images(im, seed=9)
    assert vae.encode_args[-1] == ((64, 64), [9, 9], [0, 1])
    assert torch.equal(a, CE.posterior(CE.fake_moments(im), CE.SCALE, [9, 9], [0, 1]).float())
    torch.manual_seed(3)
    vae.encode_images(im)
    torch.manual_seed(3)
    drawn = int(torch.randint(0, 2 ** 63 - 1, (1,), dtype=torch.int64).item())
    assert vae.encode_args[-1][1] == [drawn, drawn]
    with pytest.raises(ValueError, match="seed"):
        vae.encode_images(im, seed=2 ** 64)
    with pytest.raises(ValueError, match="uint8"):
        vae.encode_images(im.float(), seed=1)
    with pytest.raises(ValueError, match="multiple of 8"):
        vae.encode_images(im[:, :60], seed=1)


def test_seed_resolution_order(diffusion, torch_kernels):
    """Unseeded init_image requests draw their seeds with the x_init and DDIM eta > 0 requests, in request order, when
    sample_requests starts or at submit; the result equals the run with those seeds given."""
    S = 10
    reqs = [replace(_req(10, S), init_image=_img(10), strength=0.6), _req(11, S),
            replace(_req(12, S), x_init=torch.randn((1, 4, 64, 64), generator=torch.Generator().manual_seed(1)),
                    strength=0.5),
            replace(_req(13, S), sampler="ddim", eta=0.5), replace(_req(14, S), init_image=_img(14), strength=0.4)]
    torch.manual_seed(77)
    draws = [int(torch.randint(0, 2 ** 63 - 1, (1,), dtype=torch.int64).item()) for _ in range(4)]
    seeded = [replace(r, seed=s) for r, s in zip([reqs[0], reqs[2], reqs[3], reqs[4]], draws)]
    seeded = [seeded[0], reqs[1], seeded[1], seeded[2], seeded[3]]
    vae, model = CE.FakeAutoencoder(), FakeUNet()  # (building the fake draws from the default generator)
    torch.manual_seed(77)
    got = sample_requests(model, diffusion, [_fresh(r) for r in reqs], S, autoencoder=vae)
    assert [a[1] for a in vae.encode_args] == [[draws[0], draws[3]]]
    want = sample_requests(FakeUNet(), diffusion, [_fresh(r) for r in seeded], S, autoencoder=CE.FakeAutoencoder())
    assert all(torch.equal(a, b) for a, b in zip(got, want))
    eng = SamplingEngine(FakeUNet(), diffusion, autoencoder=CE.FakeAutoencoder())
    torch.manual_seed(77)
    tickets = [eng.submit(_fresh(r)) for r in reqs]
    assert [st.base.seed for _, st in eng._queue] == [draws[0], 0, draws[1], draws[2], draws[3]]
    assert [t for t in tickets] == list(range(5))


# ------------------------------------------------------------------------------------------------
# batching
# ------------------------------------------------------------------------------------------------
def test_encode_images_helper_groups_and_chunks(torch_kernels):
    vae = CE.FakeAutoencoder()
    ims = [_img(1, b=1, size=64), _img(2, b=2, size=32), _img(3, b=3, size=64), _img(4, b=1, size=32),
           _img(5, b=2, size=64)]
    seeds = [11, 12, 13, 14, 15]
    got = encode_images(vae, ims, seeds, 4)
    assert vae.encode_calls == [4, 2, 3]  # 6 images of 64x64 in chunks of 4 and 2, then 3 of 32x32
    assert vae.encode_args[0] == ((64, 64), [11, 13, 13, 13], [0, 0, 1, 2])
    assert vae.encode_args[1] == ((64, 64), [15, 15], [0, 1])
    assert vae.encode_args[2] == ((32, 32), [12, 12, 14], [0, 1, 0])
    for im, s, z in zip(ims, seeds, got):
        assert torch.equal(z, CE.FakeAutoencoder().encode_images(im, seed=s))


@pytest.mark.parametrize("max_encode_batch", [8, 3])
def test_sample_requests_encodes_before_the_first_step(diffusion, torch_kernels, max_encode_batch):
    S = 10
    reqs = [replace(_req(20 + k, S), init_image=_img(20 + k), strength=0.5, seed=k) for k in range(4)]
    reqs.insert(2, _req(30, S))
    reqs[1] = replace(reqs[1], input=dict(reqs[1].input, x=torch.zeros((2, 4, 64, 64)),
                                          context=reqs[1].input["context"].expand(2, -1, -1)),
                      init_image=_img(40, b=2))  # batch 2 from two images
    vae = CE.FakeAutoencoder()
    model = FakeUNet()
    sample_requests(model, diffusion, [_fresh(r) for r in reqs], S, autoencoder=vae, max_encode_batch=max_encode_batch)
    assert sum(vae.encode_calls) == 5 and max(vae.encode_calls) <= max_encode_batch
    assert len(vae.encode_calls) == -(-5 // max_encode_batch)
    seeds = [s for a in vae.encode_args for s in a[1]]
    index = [i for a in vae.encode_args for i in a[2]]
    assert seeds == [0, 1, 1, 2, 3] and index == [0, 0, 1, 0, 0]  # request order, the batch-2 request's two images
    for r in reqs:
        assert r.x_init is None  # the caller's requests are left alone


def test_engine_encodes_in_the_admission_tick(diffusion, torch_kernels):
    """Requests admitted together are encoded together in that tick, grouped by image size; one admitted later is
    encoded in its own tick."""
    S = 10
    vae = CE.FakeAutoencoder()
    eng = SamplingEngine(FakeUNet(), diffusion, max_batch=8, buckets=None, autoencoder=vae, max_encode_batch=2,
                         max_live_images=8)
    big = [replace(_req(50 + k, S), init_image=_img(50 + k), strength=0.5, seed=50 + k) for k in range(3)]
    small = replace(_req(60, S, size=32), init_image=_img(60, size=256), strength=0.5, seed=60)
    late = replace(_req(70, S), init_image=_img(70), strength=0.5, seed=70)
    for r in [big[0], small, big[1], big[2], late]:  # 2 images each with CFG: the last waits for room
        eng.submit(_fresh(r))
    eng.step()
    assert vae.encode_calls == [2, 1, 1]
    assert [a[0] for a in vae.encode_args] == [(512, 512), (512, 512), (256, 256)]
    assert [a[1] for a in vae.encode_args] == [[50, 51], [52], [60]]
    while eng.queued:
        n = len(vae.encode_calls)
        eng.step()
    assert vae.encode_calls[n:] == [1] and vae.encode_args[-1][1] == [70]
    eng.drain()


# ------------------------------------------------------------------------------------------------
# init_image == x_init = encode_images(init_image, seed=seed)
# ------------------------------------------------------------------------------------------------
def _mix(S):
    """init_image PLMS, DDIM at eta 0.7 (batch 2 from one image), DPM-Solver++(2M) and Multi-instance requests, an
    x_init request and plain PLMS / DDIM requests; some ask for images."""
    g = torch.Generator().manual_seed(5)
    b2 = _req(81, S)
    b2 = replace(b2, input=dict(b2.input, x=torch.randn((2, 4, 64, 64), generator=g),
                                context=b2.input["context"].expand(2, -1, -1)))
    return [
        replace(_req(80, S), init_image=_img(80), strength=0.6, seed=21, output="image"),
        replace(b2, sampler="ddim", eta=0.7, init_image=_img(81), strength=0.35, seed=22),
        replace(_req(82, S), sampler="dpmpp_2m", init_image=_img(82), strength=0.5, seed=23),
        replace(_req(83, S, n=2, mis=0.9), init_image=_img(83), strength=0.9, seed=24, output="image"),
        replace(_req(84, S), x_init=torch.randn((1, 4, 64, 64), generator=g), strength=0.5, seed=25),
        _req(85, S),
        replace(_req(86, S), sampler="ddim", eta=0.5, seed=26, output="image"),
    ]


def _as_x_init(reqs):
    vae = CE.FakeAutoencoder()
    return [replace(r, init_image=None, x_init=vae.encode_images(r.init_image, seed=r.seed))
            if r.init_image is not None else r for r in reqs]


def test_sample_requests_init_image_equals_x_init(diffusion, torch_kernels):
    S = 10
    reqs = _mix(S)
    vae = CE.FakeAutoencoder()
    got = sample_requests(FakeUNet(), diffusion, [_fresh(r) for r in reqs], S, max_batch=8, autoencoder=vae,
                          max_encode_batch=3)
    want = sample_requests(FakeUNet(), diffusion, [_fresh(r) for r in _as_x_init(reqs)], S, max_batch=8,
                           autoencoder=CE.FakeAutoencoder())
    assert vae.encode_calls == [3, 1]
    for k, (a, b) in enumerate(zip(got, want)):
        assert torch.equal(a, b), k
    assert got[0].dtype == torch.uint8 and got[1].shape == (2, 4, 64, 64)


def test_engine_init_image_equals_x_init(diffusion, torch_kernels):
    S = 10
    reqs = _mix(S)
    ticks = [0, 0, 1, 2, 2, 3, 5]

    def drive(rs, vae):
        eng = SamplingEngine(FakeUNet(), diffusion, max_batch=8, buckets=(2, 4, 8), autoencoder=vae, max_encode_batch=2)
        by_ticket, done, tick = {}, {}, 0
        while len(done) < len(rs):
            for j, t in enumerate(ticks):
                if t == tick:
                    by_ticket[eng.submit(_fresh(rs[j]))] = j
            for ticket, x in eng.step().items():
                done[by_ticket[ticket]] = x
            tick += 1
        return [done[j] for j in range(len(rs))]
    vae = CE.FakeAutoencoder()
    got = drive(reqs, vae)
    want = drive(_as_x_init(reqs), CE.FakeAutoencoder())
    assert vae.encode_calls == [2, 1, 1]  # ticks 0 (two requests), 1, 2
    for k, (a, b) in enumerate(zip(got, want)):
        assert torch.equal(a, b), k


def test_image_output_feeds_init_image(diffusion, torch_kernels):
    """An output="image" result as the next request's init_image: the refinement loop, image in and image out."""
    S = 10
    vae = CE.FakeAutoencoder()
    first = replace(_req(90, S), output="image")
    img = sample_requests(FakeUNet(), diffusion, [_fresh(first)], S, autoencoder=vae)[0]
    assert img.dtype == torch.uint8 and img.shape == (1, 512, 512, 3)
    again = replace(_req(91, S), init_image=img, strength=0.3, seed=4, output="image")
    got = sample_requests(FakeUNet(), diffusion, [_fresh(again)], S, autoencoder=vae)[0]
    want = sample_requests(FakeUNet(), diffusion, [_fresh(r) for r in _as_x_init([again])], S, autoencoder=vae)[0]
    assert torch.equal(got, want) and got.shape == img.shape
