#!/usr/bin/env python
"""Serving benchmark: a seeded Poisson arrival trace of sampling requests replayed against three arms, alternated:

  engine      SamplingEngine (continuous batching), fed in wall-clock time: a request is submitted once it arrived;
  waves       sample_requests in waves: each wave takes every request that has arrived and waits, grouped by S;
  sequential  every request through its own sampler, one after another in arrival order.

Trace: --requests one-image 512x512 requests (latent 64x64) with n in {1, 2, 4, 8, 12, 16, 30} box instances (cycled,
shuffled by the seed); most use the Multi-instance Sampler at mis 0.36, every 6th plain PLMS, every 5th S = --steps // 2
instead of --steps; CFG 7.5, alpha [0.8, 0, 0.2]; fp16, seeded synthetic weights and inputs.  Arrivals are Poisson at
--load times the single-request rate measured by the sequential warm-up pass.  Each arm runs once untimed (graph
capture, hoisted tensors), then the timed passes, one per load.

Prints one JSON line: per load and arm requests/s over the trace, latency (arrival to result) p50 / p95 / max, the
graphs the engine captured, torch.cuda.max_memory_reserved, the relative L2 of each latent against the sequential arm,
and the card name, power limit and SM clocks (bench.ClockSampler).

  python tools/bench_serving.py [--requests 24] [--steps 50] [--load 0.5,1.0] [--max-batch 32] [--share-pool]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time
from functools import partial

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

N_INST = (1, 2, 4, 8, 12, 16, 30)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=24)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--load", default="0.5,1.0", help="arrival rate(s) as multiples of the single-request rate")
    ap.add_argument("--max-batch", type=int, default=32)
    ap.add_argument("--share-pool", action="store_true", help="the engine's graphs share one memory pool")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_serving.py: no CUDA device (there is no CPU path)")

    from bench import ClockSampler
    from bench_requests import gpu_info
    from instancediffusion_b200 import synthetic
    from instancediffusion_b200.ldm.models.diffusion.batched import Request, sample_requests
    from instancediffusion_b200.ldm.models.diffusion.engine import SamplingEngine
    from instancediffusion_b200.ldm.models.diffusion.ldm import LatentDiffusion
    from instancediffusion_b200.ldm.models.diffusion.plms import PLMSSampler
    from instancediffusion_b200.ldm.models.diffusion.plms_instance import PLMSSamplerInst
    from instancediffusion_b200.utils.model import alpha_generator, set_alpha_scale
    from instancediffusion_b200.weights import build_unet

    device = torch.device("cuda:0")
    model = build_unet("box", device, seed=0)
    sd_conv = torch.load(os.path.join(ROOT, "tests", "golden", "sd15_first_conv.pt"), map_location="cpu")
    model.restore_first_conv_from_SD = lambda: (None if getattr(model, "_first_conv_restored", False)
                                                else model.set_sd_first_conv(sd_conv))
    model.restore_first_conv_from_SD()  # the SD1.5 conv weights are known to the per-image conv from the start
    model.undo_first_conv_restore()
    diffusion = LatentDiffusion(linear_start=0.00085, linear_end=0.012, timesteps=1000).to(device)
    gti = model.grounding_tokenizer_input
    rng = np.random.default_rng(args.seed)
    ns = [N_INST[k % len(N_INST)] for k in range(args.requests)]
    rng.shuffle(ns)
    agen = partial(alpha_generator, type=[0.8, 0.0, 0.2])
    base = []
    for k, n in enumerate(ns):
        plain = k % 6 == 5
        S = args.steps // 2 if k % 5 == 4 else args.steps
        inputs, uc = synthetic.make_sampler_inputs(gti, 1, n, 700 + k, "box", mis=not plain, device=device)
        base.append(Request(input=inputs, uc=uc, guidance_scale=7.5, alpha_generator_func=agen,
                            mis=0.0 if plain else 0.36, shape=(1, 4, 64, 64), S=S))

    def fresh(r):
        if isinstance(r.input, list):
            x = r.input[0]["x"].clone()
            return Request(**{**r.__dict__, "input": [dict(i, x=x) for i in r.input]})
        return Request(**{**r.__dict__, "input": dict(r.input, x=r.input["x"].clone())})

    def reset():
        model.undo_first_conv_restore()
        set_alpha_scale(model, 1)

    def wait_until(t0, t):
        dt = t - (time.perf_counter() - t0)
        if dt > 0:
            time.sleep(dt)

    def sequential(arrivals):
        done, out, t0 = {}, {}, time.perf_counter()
        for j in np.argsort(arrivals, kind="stable"):
            wait_until(t0, arrivals[j])
            r = fresh(base[j])
            reset()
            kw = dict(alpha_generator_func=r.alpha_generator_func, set_alpha_scale=set_alpha_scale)
            s = PLMSSamplerInst(diffusion, model, mis=r.mis, **kw) if isinstance(r.input, list) else PLMSSampler(diffusion, model, **kw)
            out[j] = s.sample(S=r.S, shape=r.shape, input=r.input, uc=r.uc, guidance_scale=r.guidance_scale)
            torch.cuda.synchronize()
            done[j] = time.perf_counter() - t0
        return done, out, {}

    def waves(arrivals):
        done, out, t0 = {}, {}, time.perf_counter()
        order = list(np.argsort(arrivals, kind="stable"))
        while order:
            now = time.perf_counter() - t0
            ready = [j for j in order if arrivals[j] <= now]
            if not ready:
                wait_until(t0, arrivals[order[0]])
                continue
            for S in sorted({base[j].S for j in ready}, reverse=True):
                group = [j for j in ready if base[j].S == S]
                reset()
                res = sample_requests(model, diffusion, [fresh(base[j]) for j in group], S, max_batch=args.max_batch)
                torch.cuda.synchronize()
                t = time.perf_counter() - t0
                for j, x in zip(group, res):
                    done[j], out[j] = t, x
            order = [j for j in order if j not in done]
        return done, out, {}

    def engine(arrivals):
        reset()
        eng = SamplingEngine(model, diffusion, max_batch=args.max_batch, share_graph_pool=args.share_pool)
        done, out, tickets, t0 = {}, {}, {}, time.perf_counter()
        order = list(np.argsort(arrivals, kind="stable"))
        while len(done) < len(base):
            now = time.perf_counter() - t0
            while order and arrivals[order[0]] <= now:
                j = order.pop(0)
                tickets[eng.submit(fresh(base[j]))] = j
            if not eng.live and not eng.queued:
                wait_until(t0, arrivals[order[0]])
                continue
            res = eng.step()
            if res:
                torch.cuda.synchronize()
                t = time.perf_counter() - t0
                for ticket, x in res.items():
                    done[tickets[ticket]], out[tickets[ticket]] = t, x
        return done, out, {"graphs_captured": eng.graphs_captured, "forwards": eng.forwards,
                           "padded_images": eng.padded_images}

    arms = {"engine": engine, "waves": waves, "sequential": sequential}
    zero = np.zeros(len(base))
    t = time.perf_counter()
    sequential(zero)  # warm-up of the sequential arm; it also measures the single-request rate
    single_rate = len(base) / (time.perf_counter() - t)
    graphs0 = len(model._graphs)
    torch.cuda.reset_peak_memory_stats()
    warm_engine = engine(zero)[2]  # graph capture of the engine's forwards
    engine_reserved = torch.cuda.max_memory_reserved()
    warm_engine["graphs"] = len(model._graphs) - graphs0
    waves(zero)

    result = {}
    for load in [float(v) for v in args.load.split(",")]:
        gaps = np.random.default_rng(args.seed + 1).exponential(1.0 / (load * single_rate), len(base))
        arrivals = np.cumsum(gaps) - gaps[0]
        per, outs = {}, {}
        for name, fn in arms.items():
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            with ClockSampler(0) as clk:
                done, out, extra = fn(arrivals)
            lat = np.array([done[j] - arrivals[j] for j in range(len(base))])
            span = max(done.values()) - arrivals.min()
            per[name] = {"requests_per_s": len(base) / span, "latency_p50_s": float(np.percentile(lat, 50)),
                         "latency_p95_s": float(np.percentile(lat, 95)), "latency_max_s": float(lat.max()),
                         "max_memory_reserved_gib": torch.cuda.max_memory_reserved() / 2 ** 30, "clocks": clk.summary(),
                         **extra}
            outs[name] = {j: x.float().cpu() for j, x in out.items()}
        for name in ("engine", "waves"):
            per[name]["latent_rel_l2_vs_sequential"] = [
                ((outs[name][j] - outs["sequential"][j]).norm() / outs["sequential"][j].norm()).item() for j in range(len(base))]
        result[str(load)] = per
    line = {
        "workload": f"{len(base)} requests x 1 image 512x512, n={ns}, MIS 0.36 (every 6th plain PLMS), S={args.steps} "
                    f"(every 5th S={args.steps // 2}), CFG 7.5, alpha [0.8, 0, 0.2], Poisson arrivals, fp16",
        "gpu": gpu_info(), "max_batch": args.max_batch, "share_graph_pool": args.share_pool,
        "single_request_rate_per_s": single_rate,
        "engine_warmup": {**warm_engine, "max_memory_reserved_gib": engine_reserved / 2 ** 30},
        "graphs_total": len(model._graphs), "loads": result,
    }
    print(json.dumps(line))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(line, fh, indent=1)


if __name__ == "__main__":
    main()
