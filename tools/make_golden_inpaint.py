"""Generate tests/golden/inpaint.pt: the latents of the reference's own, unmodified PLMSSampler.sample and
DDIMSampler.sample (eta = 0) with mask / x0 on the CPU in fp32, for the cases of tests/cases_inpaint.py, on the seeded
UNet of tests/cases.py UNET_CASE.  Needs a reference checkout ($IDIFF_REF, see oracle/ref_harness.py):

    python tools/make_golden_inpaint.py

Each case is the strength-1 inpainting request of the project's drivers: input["x"] is x_init noised at the first
timestep with the image-to-image start noise (tests/cases_img2img.py), mask is the latent keep mask of the case's pixel
box and x0 = x_init.  The reference diffusion's q_sample is wrapped to pass its own `noise=` argument the seeded blend
stream (tests/cases_noise.py INPAINT at the step's timestep) in place of torch.randn_like; the sampler loops are
not edited.  Only the latents are written.
"""
from __future__ import annotations

import os
import sys
import time
from functools import partial

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests"))
GOLDEN = os.path.join(REPO, "tests", "golden")

import cases  # noqa: E402
import cases_img2img as CI  # noqa: E402
import cases_inpaint as CP  # noqa: E402
import cases_noise as CN  # noqa: E402
from oracle import ref_harness, torch_oracle  # noqa: E402
from instancediffusion_b200 import synthetic  # noqa: E402


def case_tensors(sc):
    """(x_init, keep, x_start) of a case on the CPU: x_init (batch, 4, 64, 64) from src_seed, the keep mask of its box
    and the strength-1 start latent."""
    b = sc["batch"]
    x_init = torch.randn((b, 4, 64, 64), generator=torch.Generator().manual_seed(sc["src_seed"]))
    keep = CP.keep_of(CP.box_mask(1, 512, sc["box"]))
    _, x_start = CI.start_latent(x_init, sc["S"], 1.0, sc["seed"], (b, 4, 64, 64))
    return x_init, keep, x_start


def main():
    torch.set_num_threads(os.cpu_count())
    ref = ref_harness.import_reference()
    from ldm.models.diffusion.ddim import DDIMSampler  # the reference's modules (its root is first on sys.path)
    from ldm.models.diffusion.plms import PLMSSampler
    spec = cases.UNET_CASE
    t0 = time.time()
    model = ref_harness.build_ref_unet(ref, spec["flavor"], spec["weight_seed"])
    print(f"reference UNet built in {time.time() - t0:.1f}s", flush=True)
    diffusion = ref.LatentDiffusion(linear_start=0.00085, linear_end=0.012, timesteps=1000)
    q_sample = diffusion.q_sample
    setter = partial(ref_harness.set_alpha_scale, ref)
    out = {}
    for name, sc in CP.INPAINT_CASES.items():
        if hasattr(model, "first_conv_state_dict"):  # undo the previous case's swap to the SD1.5 conv
            conv = torch.nn.Conv2d(4, 320, 3, padding=1)
            conv.load_state_dict(model.first_conv_state_dict)
            model.input_blocks[0][0] = conv

        def seeded(x_start, t, seed=sc["seed"]):
            tt = int(t.reshape(-1)[0])
            z = torch.from_numpy(CN.normals(seed, CN.INPAINT, tt, x_start.numel())).view_as(x_start).float()
            return q_sample(x_start, t, noise=z)
        diffusion.q_sample = seeded
        agen = partial(torch_oracle.alpha_schedule, alpha_type=sc["alpha_type"])
        inputs, uc = synthetic.make_sampler_inputs(model.grounding_tokenizer_input, sc["batch"], sc["n"],
                                                   sc["input_seed"], "box", mis=False)
        x_init, keep, x_start = case_tensors(sc)
        inputs["x"] = x_start
        kind = PLMSSampler if sc["sampler"] == "plms" else DDIMSampler
        sampler = kind(diffusion, model, alpha_generator_func=agen, set_alpha_scale=setter)
        t = time.time()
        x = sampler.sample(S=sc["S"], shape=(sc["batch"], 4, 64, 64), input=inputs, uc=uc,
                           guidance_scale=sc["guidance"], mask=keep.float()[:, None], x0=x_init)
        out[name] = x.float().contiguous()
        print(f"  {name}: {time.time() - t:.1f}s absmax={x.abs().max():.3f} finite={bool(torch.isfinite(x).all())} "
              f"kept cells {int(keep.sum())}/{keep.numel()}", flush=True)
    diffusion.q_sample = q_sample
    torch.save(out, os.path.join(GOLDEN, "inpaint.pt"))


if __name__ == "__main__":
    main()
