#!/usr/bin/env python
"""DPM-Solver++(2M) against the other samplers: config-2-shaped requests (batch 4, 512x512 / latent 64x64, 8 box
instances, CFG 7.5, alpha schedule [0.8, 0, 0.2], fp16, seeded synthetic weights and inputs) through `sample_requests`
in four arms: PLMS S = 50, DDIM S = 50 (eta 0), DPM-Solver++(2M) S = 20 and S = 25.

Reports, read in the same run as the card's name and power limit:
  * per arm: UNet forwards (counted by wrapping the model's forward_batched) and images/s over --reps alternated timed
    passes (CUDA events);
  * the update kernel at batch 4 (65 536 fp32 elements, CFG, with x0_prev) against idiff_ddim_update (eta 0): CUDA
    events around the replay of a CUDA graph of --launches launches of one kernel, per launch, alternated;
  * a labelled proxy, NOT image quality: each arm's relative L2 distance to a converged solution of the same ODE on
    the seeded weights, and that of DDIM at S = 20 and 25 and DPM-Solver++ at S = 50 for equal step counts.  The ODE is
    that of the same request without the alpha schedule (one fuser scale and first conv throughout); the converged
    solution is DDIM at S = 500 from the same start noise at the arm's first timestep (the
    'uniform' grids start at 981 for S = 50, 961 for S = 25 and 951 for S = 20, all on the S = 500 grid), to the same
    end point alphas_cumprod[0].

  python tools/bench_dpm.py [--reps 3] [--launches 500] [--out results/dpm.json]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
from functools import partial

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

ARMS = (("plms", 50), ("ddim", 50), ("dpmpp_2m", 20), ("dpmpp_2m", 25))
BATCH, N_INST, GUIDANCE = 4, 8, 7.5
# the proxy also runs the solvers at each other's step counts
PROXY_ARMS = ARMS + (("ddim", 20), ("ddim", 25), ("dpmpp_2m", 50))
CONVERGED_S = 500


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--launches", type=int, default=500)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_dpm.py: no CUDA device (there is no CPU path)")

    from bench_requests import gpu_info
    from instancediffusion_b200 import ops, synthetic
    from instancediffusion_b200.ldm.models.diffusion.batched import Request, sample_requests
    from instancediffusion_b200.ldm.models.diffusion.ddim import DDIMSampler
    from instancediffusion_b200.ldm.models.diffusion.dpm_solver import dpmpp2m_coefs
    from instancediffusion_b200.ldm.models.diffusion.ldm import LatentDiffusion
    from instancediffusion_b200.ldm.modules.diffusionmodules.util import make_ddim_timesteps
    from instancediffusion_b200.utils.model import alpha_generator, set_alpha_scale
    from instancediffusion_b200.weights import build_unet

    info_before = gpu_info()
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

    counts = {"forwards": 0}
    inner = model.forward_batched

    def counting(inputs, *a, **k):
        counts["forwards"] += 1
        return inner(inputs, *a, **k)
    model.forward_batched = counting

    def reset():
        model.undo_first_conv_restore()
        set_alpha_scale(model, 1)

    def run(sampler, S, schedule=True):
        reset()
        req = Request(input=dict(inp, x=x_noise.clone()), uc=uc, guidance_scale=GUIDANCE, shape=shape, sampler=sampler,
                      alpha_generator_func=agen if schedule else None)
        out = sample_requests(model, diffusion, [req], S, max_batch=2 * BATCH)[0]
        reset()
        return out

    # 1. end to end
    for sampler, S in ARMS:  # warm-up: graph capture, hoisted tensors
        run(sampler, S)
    torch.cuda.synchronize()
    runs = {f"{s}@{S}": [] for s, S in ARMS}
    forwards = {}
    for _ in range(args.reps):
        for sampler, S in ARMS:
            key = f"{sampler}@{S}"
            counts["forwards"] = 0
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            torch.cuda.synchronize()
            ev[0].record()
            run(sampler, S)
            ev[1].record()
            torch.cuda.synchronize()
            t = ev[0].elapsed_time(ev[1]) * 1e-3
            forwards[key] = counts["forwards"]
            runs[key].append({"seconds": t, "images_per_s": BATCH / t})

    # 2. the update kernels at batch 4
    n = BATCH * 4 * 64 * 64
    g = torch.Generator().manual_seed(3)
    x, e_c, e_u, x0_prev = (torch.randn(n, generator=g).to(device) for _ in range(4))
    x_out, x0_out = torch.empty_like(x), torch.empty_like(x)
    a_t, a_n = float(np.float32(0.30212)), float(np.float32(0.61768))
    c = dpmpp2m_coefs(a_t, a_n, 0.21)[:6]
    kernels = {
        "idiff_dpmpp2m_update": lambda: ops.dpmpp2m_update(x, e_c, e_u, GUIDANCE, x0_prev, *c, x0_out, x_out),
        "idiff_ddim_update": lambda: ops.ddim_update(x, e_c, e_u, GUIDANCE, a_t, a_n, 0.0, 0, 7, None, x_out),
    }
    graphs = {}
    for name, fn in kernels.items():  # --launches launches in one CUDA graph: device time, not the Python launch path
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            fn()
        torch.cuda.current_stream().wait_stream(side)
        graphs[name] = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graphs[name]):
            for _ in range(args.launches):
                fn()
        graphs[name].replay()
    kernel_us = {k: [] for k in kernels}
    for _ in range(args.reps):
        for name, graph in graphs.items():
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            torch.cuda.synchronize()
            ev[0].record()
            graph.replay()
            ev[1].record()
            torch.cuda.synchronize()
            kernel_us[name].append(ev[0].elapsed_time(ev[1]) * 1e3 / args.launches)
    del graphs

    # 3. the proxy: distance to a converged solution of the same ODE (no alpha schedule), not image quality
    conv_steps = np.flip(make_ddim_timesteps("uniform", CONVERGED_S, 1000))
    converged = {}

    def converged_from(t_first):
        if t_first not in converged:
            reset()
            s = DDIMSampler(diffusion, model)
            s.make_schedule(CONVERGED_S)
            k0 = int(np.nonzero(conv_steps == t_first)[0][0])
            converged[t_first] = s.ddim_sampling(shape, dict(inp, x=x_noise.clone()), uc, GUIDANCE, k0=k0).float()
            reset()
        return converged[t_first]
    proxy = {}
    for sampler, S in PROXY_ARMS:
        t_first = int(make_ddim_timesteps("uniform", S, 1000)[-1])
        ref = converged_from(t_first)
        out = run(sampler, S, schedule=False).float()
        proxy[f"{sampler}@{S}"] = {"first_timestep": t_first,
                                   "rel_l2_to_converged": ((out - ref).norm() / ref.norm()).item()}

    summary = {}
    for key, rs in runs.items():
        ips = sorted(r["images_per_s"] for r in rs)
        summary[key] = {"unet_forwards": forwards[key], "images_per_s_median": ips[len(ips) // 2],
                        "images_per_s_min": ips[0], "images_per_s_max": ips[-1]}
    base = summary["plms@50"]
    for e in summary.values():
        e["forwards_vs_plms50"] = e["unet_forwards"] / base["unet_forwards"]
        e["speed_vs_plms50"] = e["images_per_s_median"] / base["images_per_s_median"]
    line = {
        "workload": f"config2-shaped: batch {BATCH} 512x512, {N_INST} box instances, CFG {GUIDANCE}, alpha schedule "
                    "[0.8, 0, 0.2], fp16, one request through sample_requests",
        "gpu": gpu_info(), "gpu_at_start": info_before, "reps": args.reps, "summary": summary, "runs": runs,
        "update_kernel_us_batch4": {k: {"median": sorted(v)[len(v) // 2], "all": v} for k, v in kernel_us.items()},
        "proxy_not_image_quality": {
            "what": f"relative L2 to DDIM at S = {CONVERGED_S} from the same start noise at the arm's first timestep, "
                    "without the alpha schedule, on seeded synthetic weights",
            "arms": proxy},
    }
    print(json.dumps(line))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(line, fh, indent=1)


if __name__ == "__main__":
    main()
