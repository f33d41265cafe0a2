#!/usr/bin/env python
"""Cost of image-to-image sampling against sampling from noise: config-2-shaped requests (batch 4, 512x512 / latent
64x64, 8 box instances, CFG 7.5, alpha schedule [0.8, 0, 0.2], 50-step PLMS, fp16, seeded synthetic weights and
inputs) at strength 1.0 (plain: no x_init), 0.6 and 0.35, each through `PLMSSampler.sample()` and through
`sample_requests` (the same request alone).  x_init is the latent of a plain warm-up run, as in a polish pass.

Reports per (strength, arm): UNet forwards and images evaluated (counted by wrapping the model's forward_batched),
seconds and images/s over --reps alternated timed passes (CUDA events), the SM clock during each pass (bench.py's
ClockSampler) and the card's name and power limit.

  python tools/bench_img2img.py [--reps 3] [--steps 50] [--out results/img2img.json]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
from functools import partial

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

STRENGTHS = (1.0, 0.6, 0.35)
BATCH, N_INST, GUIDANCE = 4, 8, 7.5


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_img2img.py: no CUDA device (there is no CPU path)")

    from bench import ClockSampler
    from bench_requests import gpu_info
    from instancediffusion_b200 import synthetic
    from instancediffusion_b200.ldm.models.diffusion.batched import Request, sample_requests
    from instancediffusion_b200.ldm.models.diffusion.ldm import LatentDiffusion
    from instancediffusion_b200.ldm.models.diffusion.plms import PLMSSampler
    from instancediffusion_b200.utils.model import alpha_generator, set_alpha_scale
    from instancediffusion_b200.weights import build_unet

    device = torch.device("cuda:0")
    model = build_unet("box", device, seed=0)
    sd_conv = torch.load(os.path.join(ROOT, "tests", "golden", "sd15_first_conv.pt"), map_location="cpu")
    model.restore_first_conv_from_SD = lambda: (None if getattr(model, "_first_conv_restored", False)
                                                else model.set_sd_first_conv(sd_conv))
    diffusion = LatentDiffusion(linear_start=0.00085, linear_end=0.012, timesteps=1000).to(device)
    inp, uc = synthetic.make_sampler_inputs(model.grounding_tokenizer_input, BATCH, N_INST, 900, "box", device=device)
    x_noise = inp["x"].clone()
    agen = partial(alpha_generator, type=[0.8, 0.0, 0.2])
    shape = (BATCH, 4, 64, 64)

    counts = {"forwards": 0, "images": 0}
    inner = model.forward_batched

    def counting(inputs, *a, **k):
        counts["forwards"] += 1
        counts["images"] += sum(i["x"].shape[0] for i in inputs)
        return inner(inputs, *a, **k)
    model.forward_batched = counting

    def reset():
        model.undo_first_conv_restore()
        set_alpha_scale(model, 1)

    x_init = [None]

    def kw(strength):
        return {} if strength == 1.0 else dict(x_init=x_init[0], strength=strength, seed=1234)

    def sample(strength):
        reset()
        s = PLMSSampler(diffusion, model, alpha_generator_func=agen, set_alpha_scale=set_alpha_scale)
        return s.sample(S=args.steps, shape=shape, input=dict(inp, x=x_noise.clone()), uc=uc, guidance_scale=GUIDANCE,
                        **kw(strength))

    def requests(strength):
        reset()
        req = Request(input=dict(inp, x=x_noise.clone()), uc=uc, guidance_scale=GUIDANCE, alpha_generator_func=agen,
                      shape=shape, **kw(strength))
        return sample_requests(model, diffusion, [req], args.steps, max_batch=2 * BATCH)[0]

    x_init[0] = sample(1.0).clone()  # warm-up of the plain run; its latent is the image to refine
    arms = {"sample": sample, "sample_requests": requests}
    for strength in STRENGTHS:  # warm-up: graph capture, hoisted tensors
        for fn in arms.values():
            fn(strength)
    torch.cuda.synchronize()

    runs = {f"{name}@{s}": [] for s in STRENGTHS for name in arms}
    evals, outs = {}, {}
    for _ in range(args.reps):
        for strength in STRENGTHS:
            for name, fn in arms.items():
                counts.update(forwards=0, images=0)
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
                torch.cuda.synchronize()
                with ClockSampler(0) as clk:
                    ev[0].record()
                    out = fn(strength)
                    ev[1].record()
                    torch.cuda.synchronize()
                t = ev[0].elapsed_time(ev[1]) * 1e-3
                key = f"{name}@{strength}"
                evals[key] = dict(counts)
                outs[key] = out.float().cpu()
                runs[key].append({"seconds": t, "images_per_s": BATCH / t, "clocks": clk.summary()})
    summary = {}
    for key, rs in runs.items():
        ips = sorted(r["images_per_s"] for r in rs)
        summary[key] = {"unet_forwards": evals[key]["forwards"], "images_evaluated": evals[key]["images"],
                        "images_per_s_median": ips[len(ips) // 2], "images_per_s_min": ips[0],
                        "images_per_s_max": ips[-1]}
    for name in arms:
        plain = summary[f"{name}@1.0"]
        for s in STRENGTHS:
            e = summary[f"{name}@{s}"]
            e["time_vs_plain"] = plain["images_per_s_median"] / e["images_per_s_median"]
            e["evaluations_vs_plain"] = e["images_evaluated"] / plain["images_evaluated"]
    rel = {s: ((outs[f"sample_requests@{s}"] - outs[f"sample@{s}"]).norm() / outs[f"sample@{s}"].norm()).item()
           for s in STRENGTHS}
    line = {
        "workload": f"config2-shaped: batch {BATCH} 512x512, {N_INST} box instances, {args.steps}-step PLMS, CFG "
                    f"{GUIDANCE}, fp16; image-to-image at strengths {list(STRENGTHS[1:])} from a plain run's latent",
        "gpu": gpu_info(), "reps": args.reps, "summary": summary, "runs": runs,
        "latent_rel_l2_sample_requests_vs_sample": rel,
    }
    print(json.dumps(line))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(line, fh, indent=1)


if __name__ == "__main__":
    main()
