"""`-m gpu` parity of the bf16-storage build (libidiff_b200_bf16.so; BASELINE config 3 = `bench.py --config 4`):
whole-UNet eps and sampler latents against the reference's fp32 goldens, next to the *measured* bf16 envelope --
the oracle port run on the same GPU under torch.autocast(bfloat16) against the same goldens.

The per-kernel bf16 checks are the second parametrisation of tests/test_kernels_gpu.py.

bf16 has 8 significand bits against fp16's 11: every rounding step is 8x coarser, so the bounds here are the fp16
bounds of test_parity_r2_gpu.py scaled by 8 and then set from the measured errors of the implementation; the envelope test bounds our deviation by the reference-under-autocast's own.
"""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import cases  # noqa: E402
import test_parity_r2_gpu as P  # noqa: E402  (helpers: inputs, sampler runner, flavour flags)

pytestmark = pytest.mark.gpu

# bounds: about 2x the measured bf16-storage errors
EPS_TOL_BF16 = 3e-2
LATENT_TOL_BF16 = 3.7e-2
ENVELOPE_FACTOR = 1.25
ENVELOPE_FACTOR_LATENT = 1.25


@pytest.fixture(scope="module")
def unet_bf16(cuda_device):
    from instancediffusion_b200 import ops
    from instancediffusion_b200.weights import build_unet
    ops.set_storage_dtype(torch.bfloat16)
    model = build_unet("box", cuda_device, seed=0)
    model._sd_conv = P._load("sd15_first_conv.pt")
    yield model
    ops.set_storage_dtype(torch.float16)


def test_storage_switch_is_loud(cuda_device):
    """A tensor of the other 16-bit type is rejected, never reinterpreted; the two builds report their type."""
    from instancediffusion_b200 import _lib, ops
    assert _lib.load("f16").idiff_storage_dtype() == 0 and _lib.load("bf16").idiff_storage_dtype() == 1
    a = torch.randn(128, 64, device=cuda_device)
    w = torch.randn(128, 64, device=cuda_device)
    with ops.storage(torch.float16):
        with ops.storage(torch.bfloat16):
            out = ops.gemm(a.bfloat16(), w.bfloat16())
            assert out.dtype == torch.bfloat16
            ref = a.bfloat16().float() @ w.bfloat16().float().t()
            assert ((out.float() - ref).norm() / ref.norm()).item() < 4e-3
            with pytest.raises(_lib.IdiffError):
                ops.gemm(a.half(), w.half())
        assert ops.storage_dtype() == torch.float16
        with pytest.raises(_lib.IdiffError):
            ops.gemm(a.bfloat16(), w.bfloat16())


@pytest.mark.parametrize("name", ["b4n8", "mask", "lat96"])
def test_unet_eps_bf16_vs_reference_golden(cuda_device, unet_bf16, name):
    """The bench forward (b4n8), the mask flavour (ConvNeXt tokens) and the 96x96 latent of config 4, bf16 storage."""
    from instancediffusion_b200.utils.model import set_alpha_scale
    unet = unet_bf16
    gold = P._load("unet_extra.pt")
    spec = cases.UNET_EXTRA_CASES[name]
    if name + "/eps_cond" not in gold:
        pytest.skip(f"{name} not in unet_extra.pt")
    P._set_flavor(unet.position_net, spec["flavor"])
    unet.clear_caches()
    unet.undo_first_conv_restore()
    set_alpha_scale(unet, 1)
    try:
        inp, uc, ts = P._inputs(unet, spec, cuda_device)
        cond = dict(x=inp["x"], timesteps=ts, context=inp["context"], grounding_input=inp["grounding_input"])
        for graph in (False, True):
            unet.use_cuda_graph = graph
            if spec.get("uncond"):
                e_c, e_u = unet.forward_batched([cond, dict(x=inp["x"], timesteps=ts, context=uc)])
                r_u = P._rel(e_u, gold[name + "/eps_null"])
            else:
                e_c, r_u = unet(cond), 0.0
            r_c = P._rel(e_c, gold[name + "/eps_cond"])
            print(f"[bf16 unet/{name} graph={graph}] rel_l2 cond {r_c:.3e} uncond {r_u:.3e} (tol {EPS_TOL_BF16:.0e})")
            assert r_c < EPS_TOL_BF16 and r_u < EPS_TOL_BF16, (name, r_c, r_u)
    finally:
        P._set_flavor(unet.position_net, "box")
        unet.clear_caches()
        unet.use_cuda_graph = True


def test_bf16_envelope_eps_and_latent(cuda_device, unet_bf16):
    """What bf16 arithmetic gives the reference itself: the oracle port under torch.autocast(bfloat16) on this GPU
    (cuBLAS / cuDNN kernels, fp32 norms and softmax) against the fp32 goldens, at one eps (bench batch) and the
    10-step Multi-instance latent, in the two attention realisations of test_parity_r2_gpu.py; our bf16 build must
    stay within ENVELOPE_FACTOR (eps) / ENVELOPE_FACTOR_LATENT (latent) of the worse one, and under the absolute
    bounds above."""
    from oracle import torch_oracle as TO
    from instancediffusion_b200 import synthetic
    from instancediffusion_b200.utils.model import set_alpha_scale
    from instancediffusion_b200.weights import UNIFUSION_FLAGS, synth_tensor
    import json
    unet = unet_bf16
    flags = UNIFUSION_FLAGS["box"]
    schema = json.load(open(os.path.join(P.GOLDEN, "unet_schema.json")))
    osd = {k: synth_tensor(k, tuple(s), 0).to(cuda_device) for k, s in schema.items() if "convnext" not in k}
    sd15 = {k: v.to(cuda_device) for k, v in unet._sd_conv.items()}
    report = []

    def both(fn):
        out = []
        for fused in (False, True):
            TO.FUSED_SDPA = fused
            try:
                out.append(fn())
            finally:
                TO.FUSED_SDPA = False
        return out

    spec = cases.UNET_EXTRA_CASES["b4n8"]
    gold_u = P._load("unet_extra.pt")
    inp, uc, ts = P._inputs(unet, spec, cuda_device)
    gi = inp["grounding_input"]

    def ref_eps():
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            return TO.unet_forward(osd, inp["x"], ts, inp["context"], gi, flags)
    refs = both(ref_eps)
    set_alpha_scale(unet, 1)
    unet.clear_caches()
    ours = unet(dict(x=inp["x"], timesteps=ts, context=inp["context"], grounding_input=gi))
    g = gold_u["b4n8/eps_cond"]
    report.append(("eps b4n8", P._rel(ours, g), [P._rel(r, g) for r in refs], ENVELOPE_FACTOR, EPS_TOL_BF16))

    gold_s = P._load("samplers_extra.pt")
    name = "mis_S10_n3"
    if name in gold_s:
        sc = cases.SAMPLER_EXTRA_CASES[name]
        ours = P._run_sampler(unet, sc, cuda_device)
        inputs, uc = synthetic.make_sampler_inputs(unet.grounding_tokenizer_input, sc["batch"], sc["n"], sc["seed"], "box",
                                                   mis=sc["mis"] > 0, device=cuda_device)
        inputs = inputs if isinstance(inputs, list) else [inputs]
        ngi = TO.null_grounding_input(inputs[0]["grounding_input"])

        def eval_fn(i, alpha):
            gi_ = i.get("grounding_input")
            with torch.autocast("cuda", dtype=torch.bfloat16):
                e = TO.unet_forward(osd, i["x"], i["timesteps"], i["context"], gi_ if gi_ is not None else ngi, flags,
                                    scale=float(alpha), first_conv=sd15 if alpha == 0 else None)
            return e.float()

        def ref_latent():
            with torch.no_grad():
                ins = [dict(i, x=i["x"].clone()) for i in inputs]
                return TO.plms_sample(eval_fn, ins, uc, sc["S"], sc["guidance"], sc["mis"], alpha_type=sc["alpha_type"])
        refs = both(ref_latent)
        report.append((name, P._rel(ours, gold_s[name]), [P._rel(r, gold_s[name]) for r in refs],
                       ENVELOPE_FACTOR_LATENT, LATENT_TOL_BF16))

    for what, ours_e, ref_e, fac, tol in report:
        print(f"[bf16 envelope] {what}: ours {ours_e:.3e}   reference-under-autocast(bf16) explicit {ref_e[0]:.3e} / "
              f"fused-SDPA {ref_e[1]:.3e}   ours/worse-ref {ours_e / max(ref_e):.2f}   (bound {fac}, abs {tol:.0e})")
    for what, ours_e, ref_e, fac, tol in report:
        assert ours_e <= fac * max(ref_e) and ours_e < tol, (what, ours_e, ref_e)
