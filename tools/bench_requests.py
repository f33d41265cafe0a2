#!/usr/bin/env python
"""Throughput of many independent requests: `sample_requests` (all requests advanced in lock step, forwards of up to
--max-batch images) against the same requests run one after another through their own `sample()`.

Workload: 8 requests of 1 image each (512x512, latent 64x64), Multi-instance Sampler mis 0.36 with
n = 1, 2, 4, 8, 8, 12, 16, 30 box instances, 50-step PLMS, CFG 7.5, alpha schedule [0.8, 0, 0.2] except two
requests at [0.6, 0, 0.4]; fp16, seeded synthetic weights and inputs.  One warm-up pass of each arm (CUDA graph
capture, hoisted tensors), then --reps timed passes of each, alternating, device-timed with CUDA events.  The SM clock
is sampled with nvidia-smi during each timed pass (bench.py's ClockSampler); the latents of the two arms are compared.

  python tools/bench_requests.py [--reps 2] [--max-batch 32] [--steps 50]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
from functools import partial

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N_INST = (1, 2, 4, 8, 8, 12, 16, 30)
ALPHA_06 = (3, 6)  # requests at alpha 0.6


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=10).stdout.strip()
        return out.splitlines()[0] if out else None
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--max-batch", type=int, default=32)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_requests.py: no CUDA device (there is no CPU path)")

    from bench import ClockSampler
    from instancediffusion_b200 import synthetic
    from instancediffusion_b200.ldm.models.diffusion.batched import Request, sample_requests
    from instancediffusion_b200.ldm.models.diffusion.ldm import LatentDiffusion
    from instancediffusion_b200.ldm.models.diffusion.plms_instance import PLMSSamplerInst
    from instancediffusion_b200.utils.model import alpha_generator, set_alpha_scale
    from instancediffusion_b200.weights import build_unet

    device = torch.device("cuda:0")
    model = build_unet("box", device, seed=0)
    sd_conv = torch.load(os.path.join(ROOT, "tests", "golden", "sd15_first_conv.pt"), map_location="cpu")
    model.restore_first_conv_from_SD = lambda: (None if getattr(model, "_first_conv_restored", False)
                                                else model.set_sd_first_conv(sd_conv))
    diffusion = LatentDiffusion(linear_start=0.00085, linear_end=0.012, timesteps=1000).to(device)
    gti = model.grounding_tokenizer_input
    base = []
    for k, n in enumerate(N_INST):
        inputs, uc = synthetic.make_sampler_inputs(gti, 1, n, 500 + k, "box", mis=True, device=device)
        alpha = [0.6, 0.0, 0.4] if k in ALPHA_06 else [0.8, 0.0, 0.2]
        base.append(Request(input=inputs, uc=uc, guidance_scale=7.5, alpha_generator_func=partial(alpha_generator, type=alpha),
                            mis=0.36, shape=(1, 4, 64, 64)))

    def fresh():
        out = []
        for r in base:
            x = r.input[0]["x"].clone()
            out.append(Request(**{**r.__dict__, "input": [dict(i, x=x) for i in r.input]}))
        return out

    def reset():
        model.undo_first_conv_restore()
        set_alpha_scale(model, 1)

    def sequential():
        res = []
        for r in fresh():
            reset()
            s = PLMSSamplerInst(diffusion, model, alpha_generator_func=r.alpha_generator_func,
                                set_alpha_scale=set_alpha_scale, mis=r.mis)
            res.append(s.sample(S=args.steps, shape=r.shape, input=r.input, uc=r.uc, guidance_scale=r.guidance_scale))
        return res

    def batched():
        reset()
        return sample_requests(model, diffusion, fresh(), args.steps, max_batch=args.max_batch)

    def timed(fn):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        torch.cuda.synchronize()
        with ClockSampler(0) as clk:
            ev[0].record()
            out = fn()
            ev[1].record()
            torch.cuda.synchronize()
        return ev[0].elapsed_time(ev[1]) * 1e-3, clk.summary(), out

    arms = {"sequential": sequential, "sample_requests": batched}
    for fn in arms.values():  # warm-up: graph capture, hoisted tensors
        fn()
    torch.cuda.synchronize()
    runs = {k: [] for k in arms}
    outs = {}
    for _ in range(args.reps):
        for name, fn in arms.items():
            t, clk, out = timed(fn)
            runs[name].append({"seconds": t, "requests_per_s": len(base) / t, "images_per_s": len(base) / t, "clocks": clk})
            outs[name] = [o.float().cpu() for o in out]
    rel = [((a - b).norm() / b.norm()).item() for a, b in zip(outs["sample_requests"], outs["sequential"])]
    best = {k: max(r["requests_per_s"] for r in v) for k, v in runs.items()}
    line = {
        "workload": f"{len(base)} requests x 1 image 512x512, MIS 0.36, n={list(N_INST)}, {args.steps}-step PLMS, CFG 7.5, "
                    f"alpha 0.8 (requests {list(ALPHA_06)} at 0.6), fp16",
        "gpu": gpu_info(), "max_batch": args.max_batch, "reps": args.reps, "runs": runs,
        "speedup_best": best["sample_requests"] / best["sequential"],
        "latent_rel_l2_vs_sequential": rel,
    }
    print(json.dumps(line))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(line, fh, indent=1)


if __name__ == "__main__":
    main()
