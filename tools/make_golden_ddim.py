"""Generate tests/golden/ddim.pt: the latents of the reference's own, unmodified DDIMSampler.sample (eta = 0) on the CPU
in fp32 for the cases of tests/cases_ddim.py, on the seeded UNet of tests/cases.py UNET_CASE.  Needs a reference
checkout ($IDIFF_REF, see oracle/ref_harness.py):

    python tools/make_golden_ddim.py
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
import cases_ddim  # noqa: E402
from oracle import ref_harness, torch_oracle  # noqa: E402
from instancediffusion_b200 import synthetic  # noqa: E402


def main():
    torch.set_num_threads(os.cpu_count())
    ref = ref_harness.import_reference()
    from ldm.models.diffusion.ddim import DDIMSampler  # the reference's module (its root is first on sys.path)
    spec = cases.UNET_CASE
    t0 = time.time()
    model = ref_harness.build_ref_unet(ref, spec["flavor"], spec["weight_seed"])
    print(f"reference UNet built in {time.time() - t0:.1f}s", flush=True)
    diffusion = ref.LatentDiffusion(linear_start=0.00085, linear_end=0.012, timesteps=1000)
    setter = partial(ref_harness.set_alpha_scale, ref)
    out = {}
    for name, sc in cases_ddim.DDIM_CASES.items():
        if hasattr(model, "first_conv_state_dict"):  # undo the previous case's swap to the SD1.5 conv
            conv = torch.nn.Conv2d(4, 320, 3, padding=1)
            conv.load_state_dict(model.first_conv_state_dict)
            model.input_blocks[0][0] = conv
        agen = partial(torch_oracle.alpha_schedule, alpha_type=sc["alpha_type"])
        inputs, uc = synthetic.make_sampler_inputs(model.grounding_tokenizer_input, sc["batch"], sc["n"], sc["seed"],
                                                   "box", mis=False)
        sampler = DDIMSampler(diffusion, model, alpha_generator_func=agen, set_alpha_scale=setter)
        t = time.time()
        x = sampler.sample(S=sc["S"], shape=(sc["batch"], 4, 64, 64), input=inputs, uc=uc, guidance_scale=sc["guidance"])
        out[name] = x.float().contiguous()
        print(f"  {name}: {time.time() - t:.1f}s absmax={x.abs().max():.3f} finite={bool(torch.isfinite(x).all())}",
              flush=True)
    torch.save(out, os.path.join(GOLDEN, "ddim.pt"))


if __name__ == "__main__":
    main()
