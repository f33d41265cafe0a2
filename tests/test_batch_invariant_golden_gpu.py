"""`-m gpu` batch-invariant mode against the reference goldens: the UNet eps (unet.pt, unet_extra.pt, in fp16 and
bf16 storage), the sampler latents (samplers.pt, through the drop-in samplers and through sample_requests) and the
VAE decode (vae.pt), each with the mode on, under the existing tests' own fixtures and bounds -- those tests are
called as they are, once per mode, so the default-mode relative L2 is printed next to the invariant one.  The two
modes' eps may differ (different tile widths and reduction orders) by no more than the case's bound."""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import cases  # noqa: E402
import test_bf16_gpu as B16  # noqa: E402
import test_modules_gpu as TM  # noqa: E402
import test_parity_r2_gpu as P  # noqa: E402
import test_vae_gpu as V  # noqa: E402

pytestmark = pytest.mark.gpu
MODES = (("default", False), ("invariant", True))


@pytest.fixture(scope="module")
def unet(cuda_device):
    from instancediffusion_b200.weights import build_unet
    model = build_unet("box", cuda_device, seed=0)
    model._sd_conv = TM._load("sd15_first_conv.pt")
    # the reference reads the SD1.5 first conv from the cwd at alpha == 0; the same tensors are a fixture
    model.restore_first_conv_from_SD = lambda: (None if getattr(model, "_first_conv_restored", False)
                                                else model.set_sd_first_conv(model._sd_conv))
    yield model
    model.use_cuda_graph = True


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


def _in_both_modes(run):
    """run() with the mode off, then on; its printed lines are headed by the mode."""
    from instancediffusion_b200 import ops
    out = {}
    try:
        for name, on in MODES:
            ops.set_batch_invariant(on)
            print(f"--- {name} mode ---")
            out[name] = run()
    finally:
        ops.set_batch_invariant(False)
    return out


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / b.norm()).item()


def _mode_difference(eps, what, tol):
    r = _rel(eps["invariant"], eps["default"])
    print(f"[{what}] invariant vs default eps rel_l2 {r:.3e} (tol {tol:.0e})")
    assert r < tol, (what, r)


def test_unet_eps_invariant_vs_golden(cuda_device, unet):
    """unet.pt: eps_cond, eps_null, eps_alpha0 and the batched pair, bounds of test_modules_gpu."""
    _in_both_modes(lambda: TM.test_unet_eps_matches_reference_golden(cuda_device, unet))
    inp, uc, ts = TM._unet_inputs(unet, cuda_device)
    gi = inp["grounding_input"]
    unet.use_cuda_graph = False
    try:
        eps = _in_both_modes(lambda: unet.forward_batched([dict(x=inp["x"], timesteps=ts, context=inp["context"],
                                                                grounding_input=gi),
                                                           dict(x=inp["x"], timesteps=ts, context=uc)]))
    finally:
        unet.use_cuda_graph = True
    for k, what in enumerate(("cond", "null")):
        _mode_difference({m: e[k] for m, e in eps.items()}, f"unet/eps_{what}", 4e-3)


def _extra_eps(unet, dev, name):
    spec = cases.UNET_EXTRA_CASES[name]
    P._set_flavor(unet.position_net, spec["flavor"])
    unet.clear_caches()
    unet.use_cuda_graph = False
    try:
        inp, uc, ts = P._inputs(unet, spec, dev)
        return unet(dict(x=inp["x"], timesteps=ts, context=inp["context"], grounding_input=inp["grounding_input"]))
    finally:
        P._set_flavor(unet.position_net, "box")
        unet.clear_caches()
        unet.use_cuda_graph = True


@pytest.mark.parametrize("name", list(cases.UNET_EXTRA_CASES))
def test_unet_extra_invariant_vs_golden(cuda_device, unet, name):
    """unet_extra.pt with the bounds of test_parity_r2_gpu."""
    _in_both_modes(lambda: P.test_unet_eps_extra_vs_reference_golden(cuda_device, unet, name))
    _mode_difference(_in_both_modes(lambda: _extra_eps(unet, cuda_device, name)), f"unet_extra/{name}", P.EPS_TOL)


@pytest.mark.parametrize("name", ["b4n8", "mask", "lat96"])
def test_unet_bf16_invariant_vs_golden(cuda_device, unet, name):
    """The bf16-storage cases with the bounds of test_bf16_gpu."""
    from instancediffusion_b200 import ops
    with ops.storage(torch.bfloat16):
        _in_both_modes(lambda: B16.test_unet_eps_bf16_vs_reference_golden(cuda_device, unet, name))
        eps = _in_both_modes(lambda: _extra_eps(unet, cuda_device, name))
    _mode_difference(eps, f"bf16 unet/{name}", B16.EPS_TOL_BF16)


@pytest.mark.parametrize("name", list(cases.SAMPLER_CASES))
def test_sampler_invariant_vs_golden(cuda_device, unet, name):
    """samplers.pt through the drop-in samplers and through sample_requests, bounds of test_modules_gpu."""
    from functools import partial
    from instancediffusion_b200 import synthetic
    from instancediffusion_b200.ldm.models.diffusion.batched import Request, sample_requests
    from instancediffusion_b200.ldm.models.diffusion.ldm import LatentDiffusion
    from instancediffusion_b200.utils.model import alpha_generator, set_alpha_scale
    _in_both_modes(lambda: TM.test_sampler_latent_vs_reference_golden(cuda_device, unet, name))
    gold = TM._load("samplers.pt")
    sc = cases.SAMPLER_CASES[name]
    diffusion = LatentDiffusion(linear_start=0.00085, linear_end=0.012, timesteps=1000).to(cuda_device)

    def run():
        inputs, uc = synthetic.make_sampler_inputs(unet.grounding_tokenizer_input, sc["batch"], sc["n"], sc["seed"],
                                                   "box", mis=sc["mis"] > 0, device=cuda_device)
        req = Request(input=inputs, uc=uc, guidance_scale=sc["guidance"], mis=sc["mis"], S=sc["S"],
                      alpha_generator_func=partial(alpha_generator, type=sc["alpha_type"]),
                      shape=(sc["batch"], 4, 64, 64))
        try:
            x = sample_requests(unet, diffusion, [req], sc["S"])[0]
        finally:
            unet.undo_first_conv_restore()
            set_alpha_scale(unet, 1)
        TM._report(x, gold[name], f"sample_requests/{name}", 7.2e-3, 8.7e-3)
    _in_both_modes(run)


@pytest.mark.parametrize("name", [n for n, s in cases.VAE_CASES.items() if s["kind"] == "decode"])
def test_vae_decode_invariant_vs_golden(cuda_device, vae, name):
    """vae.pt decode, bounds of test_vae_gpu."""
    _in_both_modes(lambda: V.test_vae_decode_matches_reference_golden(cuda_device, vae, name))
